package edu.nju.pasalab.marlin.matrix

import breeze.linalg.{DenseMatrix => BDM, DenseVector => BDV}

/**
 * The per-partition bodies of DenseVecMatrix that leave the JVM (what a maintainer substitutes inside the existing
 * `mapPartitions` closures; the RDD plumbing around them stays as it is):
 *
 *  - `multiply(B: BDM[Double])` (matrix/DenseVecMatrix.scala:1660-1680): the reference packs the partition's rows into a
 *    k x rows matrix, multiplies `B.t.copy * rowsMat` with Breeze and slices the columns back into rows.  Here the rows
 *    go to the device as they are (row-major, back to back), one call computes `rows * B` with the DMMA kernel —
 *    row-major C = A * B is computed as C^T = B^T * A^T, so neither the `B.t.copy` nor the rowsMat transpose exists —
 *    and the result rows come back row-major;
 *  - the single-block ("breeze" mode) leaves of `luDecompose`, `choleskyDecompose`, `inverse`
 *    (:302 brzLU, :495 brzCholesky, :587 brzInv) and the per-block calls of the "dist" mode (:329, :349, :513, :525, :606,
 *    :617, and the triangular solves `l \ permutation`, `block * inv(u)` at :378-384) on device blocks.
 */
private[marlin] object DenseVecMatrixNative {

  /** One partition of `multiply(B: BDM[Double])`: (row id, row) pairs in, (row id, row of the product) pairs out. */
  def multiplyPartition(iter: Iterator[(Long, BDV[Double])], numCols: Int, b: BDM[Double]): Iterator[(Long, BDV[Double])] = {
    val part = iter.toArray
    val rows = part.length
    if (rows == 0) return Iterator.empty
    require(numCols == b.rows, s"Dimension mismatch during matrix-matrix multiplication: $numCols vs ${b.rows}")
    val packed = new Array[Double](rows * numCols)                 // row-major, numCols doubles per row
    var i = 0
    while (i < rows) {
      val v = part(i)._2
      if (v.stride == 1) System.arraycopy(v.data, v.offset, packed, i * numCols, numCols)
      else { var j = 0; while (j < numCols) { packed(i * numCols + j) = v(j); j += 1 } }
      i += 1
    }
    val bCol = if (!b.isTranspose && b.offset == 0 && b.majorStride == b.rows) b.data else b.copy.data   // packed column-major
    val out = new Array[Double](rows * b.cols)
    Native.matmulRowshardedHost(Ctx.get, packed, rows.toLong, numCols, bCol, b.cols, out)
    Iterator.tabulate(rows)(r => (part(r)._1, new BDV[Double](out, r * b.cols, 1, b.cols)))
  }

  /** One partition of one iteration of `lr(stepSize, iters)` (:1005-1035): the sum of the partition's per-row gradients
   *  at `weights`, as one vector (none for an empty partition).  The driver keeps its loop: `reduce(_ + _)` over the
   *  partitions, then `weights - delta * (stepSize / dataSize / math.sqrt(i))`.  Column 0 of a row is its label. */
  def lrGradientPartition(iter: Iterator[(Long, BDV[Double])], weights: BDV[Double]): Iterator[BDV[Double]] = {
    val part = iter.toArray
    val rows = part.length
    if (rows == 0) return Iterator.empty
    val numCols = weights.length
    val packed = new Array[Double](rows * numCols)                 // row-major, numCols doubles per row
    var i = 0
    while (i < rows) {
      val v = part(i)._2
      require(v.length == numCols, s"Dimension mismatch: row of ${v.length} vs $numCols weights")
      if (v.stride == 1) System.arraycopy(v.data, v.offset, packed, i * numCols, numCols)
      else { var j = 0; while (j < numCols) { packed(i * numCols + j) = v(j); j += 1 } }
      i += 1
    }
    val grad = new Array[Double](numCols)
    Native.lrGradient(Ctx.get, packed, rows, weights.toArray, grad)          // uploads, computes and frees in one call
    Iterator.single(BDV(grad))
  }

  /** brzLU(mat): (packed L\U like dgetrf, the reference's permutation array: row i of L*U is row perm(i) of mat). */
  def lu(mat: SubMatrix): (SubMatrix, Array[Int]) = {
    val work = mat.copy()
    val perm = new Array[Int](mat.rows)
    Native.lu(Ctx.get, work.handle, perm)
    (work, perm)
  }

  /** brzCholesky(mat): lower L with mat = L * L.t, strict upper triangle zero. */
  def cholesky(mat: SubMatrix): SubMatrix = {
    val work = mat.copy()
    Native.cholesky(Ctx.get, work.handle)
    work
  }

  /** brzInv(mat). */
  def inverse(mat: SubMatrix): SubMatrix = {
    val out = new SubMatrix(Native.alloc(Ctx.get, mat.rows, mat.cols, Native.F64), mat.rows, mat.cols)
    Native.inverse(Ctx.get, mat.handle, out.handle)
    out
  }

  /** computeGramianMatrix (:1464-1486) of the rows in `mat` (a row shard is a transposed view): mat.t * mat, exactly
   *  symmetric.  Partitions still combine with `+=`. */
  def gramian(mat: SubMatrix): SubMatrix = {
    val out = new SubMatrix(Native.alloc(Ctx.get, mat.cols, mat.cols, Native.F64), mat.cols, mat.cols)
    Native.gramian(Ctx.get, mat.handle, out.handle)
    out
  }

  /** The eigen step of computeSVD (:1589-1606) on a symmetric block: all eigenvalues ordered by |w| descending and the
   *  eigenvectors as columns (parallel Jacobi on the device; every mode uses it). */
  def symmetricEigen(g: SubMatrix): (Array[Double], SubMatrix) = {
    val v = new SubMatrix(Native.alloc(Ctx.get, g.rows, g.rows, Native.F64), g.rows, g.rows)
    val w = new Array[Double](g.rows)
    Native.syev(Ctx.get, g.handle, v.handle, w)
    (w, v)
  }

  /** `t \ b` for a triangular t (lower / upper, unit or explicit diagonal): solves in a copy of b. */
  def solveTriangular(t: SubMatrix, lower: Boolean, unitDiagonal: Boolean, b: SubMatrix): SubMatrix = {
    val x = b.copy()
    Native.trsm(Ctx.get, t.handle, lower, unitDiagonal, x.handle)
    x
  }

  /** `b * inv(u)` (:384) without forming the inverse: X u = b  <=>  u.t X.t = b.t, on transposed views. */
  def solveTriangularRight(b: SubMatrix, u: SubMatrix, upper: Boolean, unitDiagonal: Boolean): SubMatrix = {
    val x = b.copy()
    Native.trsm(Ctx.get, u.t.handle, upper, unitDiagonal, x.t.handle)   // the transpose of an upper factor is lower
    x
  }
}

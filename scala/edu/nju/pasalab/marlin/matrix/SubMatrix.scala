package edu.nju.pasalab.marlin.matrix

import breeze.linalg.{DenseMatrix => BDM}

/**
 * Device-resident SubMatrix: the per-block value type of BlockMatrix with the public shape of the reference's class
 * (matrix/SubMatrix.scala:6-139 — constructors from a Breeze matrix, rows / cols / isSparse, add / subtract / divide /
 * multiply overloads), holding a handle to an `mb_block` in HBM instead of a `BDM[Double]` on the heap.
 * BlockMatrix and DenseVecMatrix above it are unchanged: `block1.multiply(block2)` (BlockMatrix.scala:175) is now one
 * DMMA launch on the H100, `a.add(b)` (:177) one HBM-bound kernel.  Data crosses PCIe only when a block is built from a
 * Breeze matrix or read back through `denseBlock` (toBreeze, save).  A sparse block (`new SubMatrix(spMatrix)`) holds an
 * `mb_sparse` handle (CSC in HBM) instead: `multiply` dispatches the four sparsity pairs of the reference (:87-119) to the
 * device kernels that replace LibMatrixMult and SparseMatrix.multiply, and the scalar ops change only the stored values
 * (:52-58, 71-85, 121-129), as the reference does.
 */
class SubMatrix private[marlin] (private[marlin] val handle: Long, val rows: Int, val cols: Int,
                                 private[marlin] val sparseHandle: Long = 0L)
  extends Serializable {

  /** `new SubMatrix(denseMatrix = m)`: the Breeze record goes to HBM as it is — offset, majorStride and isTranspose are
   *  honoured by the upload, nothing is repacked on the heap. */
  def this(denseMatrix: BDM[Double]) = this(
    Native.upload(Ctx.get, denseMatrix.data, denseMatrix.offset, denseMatrix.rows, denseMatrix.cols,
      denseMatrix.majorStride, denseMatrix.isTranspose, Native.F64),
    denseMatrix.rows, denseMatrix.cols)

  /** `new SubMatrix(spMatrix = m)`: the SparseVectors flattened to CSC (SparseMatrix.toBreeze, Matrices.scala:70-104)
   *  and uploaded; unsorted or repeated row indices are rejected with IllegalArgumentException. */
  def this(spMatrix: SparseMatrix) = this(0L, spMatrix.numRows, spMatrix.numCols, SubMatrix.uploadSparse(spMatrix))

  def isSparse: Boolean = sparseHandle != 0L

  private def fresh(r: Int, c: Int): Long = Native.alloc(Ctx.get, r, c, Native.F64)

  private def sparseOp(op: Int, b: Double): SubMatrix =
    new SubMatrix(0L, rows, cols, Native.sparseValuesOp(Ctx.get, sparseHandle, op, b))

  private def requireBothDense(other: SubMatrix, op: String): Unit =
    if (isSparse || other.isSparse)
      throw new IllegalArgumentException(s"Not supported $op-operator between matrices of sparsity " +
        s"with ${this.isSparse} and ${other.isSparse}")

  /** SparseMatrix.toDense (Matrices.scala:106-119) on the device; a dense block is returned as it is. */
  private[marlin] def toDenseBlock: SubMatrix =
    if (!isSparse) this
    else { val out = fresh(rows, cols); Native.sparseToDense(Ctx.get, sparseHandle, out); new SubMatrix(out, rows, cols) }

  /** The stored CSC of a sparse block read back as the reference's SparseMatrix. */
  private[marlin] def sparseBlock: SparseMatrix = {
    require(isSparse, "sparseBlock of a dense block")
    val nnz = Native.sparseNnz(sparseHandle).toInt
    val colptr = new Array[Int](cols + 1); val rowidx = new Array[Int](nnz); val values = new Array[Double](nnz)
    Native.sparseDownload(Ctx.get, sparseHandle, colptr, rowidx, values)
    new SparseMatrix(rows, cols, Array.tabulate(cols)(j => new SparseVector(rows, rowidx.slice(colptr(j), colptr(j + 1)),
      values.slice(colptr(j), colptr(j + 1)))))
  }

  /** toBreeze / save only: reads the block back as a packed column-major Breeze matrix. */
  private[marlin] def denseBlock: BDM[Double] = {
    if (isSparse) { val d = toDenseBlock; try return d.denseBlock finally d.release() }
    val out = new Array[Double](rows * cols)
    Native.download(Ctx.get, handle, out, math.max(1, rows))
    new BDM[Double](rows, cols, out)
  }

  /** Breeze `.t`: a transposed view, no copy (used by BlockMatrix.transpose before `.copy`). */
  private[marlin] def t: SubMatrix = new SubMatrix(Native.viewT(Ctx.get, handle), cols, rows)

  def add(other: SubMatrix): SubMatrix = {
    requireBothDense(other, "add")
    val out = fresh(rows, cols); Native.add(Ctx.get, handle, other.handle, out); new SubMatrix(out, rows, cols)
  }

  def add(b: Double): SubMatrix = {
    if (isSparse) return sparseOp(0, b)
    val out = fresh(rows, cols); Native.axpb(Ctx.get, handle, 1.0, b, out); new SubMatrix(out, rows, cols)
  }

  def subtract(other: SubMatrix): SubMatrix = {
    requireBothDense(other, "subtract")
    val out = fresh(rows, cols); Native.sub(Ctx.get, handle, other.handle, out); new SubMatrix(out, rows, cols)
  }

  def subtract(b: Double): SubMatrix = {
    if (isSparse) return sparseOp(1, b)
    val out = fresh(rows, cols); Native.axpb(Ctx.get, handle, 1.0, -b, out); new SubMatrix(out, rows, cols)
  }

  def divide(b: Double): SubMatrix = {
    if (isSparse) return sparseOp(3, b)
    val out = fresh(rows, cols); Native.div(Ctx.get, handle, b, false, out); new SubMatrix(out, rows, cols)
  }

  /** The kernel seam: was `this.denseBlock * other.denseBlock` -> Breeze -> netlib dgemm, and for a sparse side
   *  LibMatrixMult.multDenseSparse / multSparseDense or SparseMatrix.multiply (:92-100); the result is dense. */
  def multiply(other: SubMatrix): SubMatrix = {
    val out = fresh(rows, other.cols)
    (isSparse, other.isSparse) match {
      case (false, false) => Native.gemm(Ctx.get, handle, other.handle, out, false)
      case (true, true) => Native.spgemm(Ctx.get, sparseHandle, other.sparseHandle, out, false)
      case (false, true) => Native.spmmDenseSparse(Ctx.get, handle, other.sparseHandle, out, false)
      case (true, false) => Native.spmmSparseDense(Ctx.get, sparseHandle, other.handle, out, false)
    }
    new SubMatrix(out, rows, other.cols)
  }

  /** `multiply(other: BDM[Double])`: the broadcast matrix is uploaded once per call site and multiplied on the device. */
  def multiply(other: BDM[Double]): SubMatrix = {
    val b = new SubMatrix(other)
    try multiply(b) finally b.release()
  }

  def multiply(b: Double): SubMatrix = {
    if (isSparse) return sparseOp(2, b)
    val out = fresh(rows, cols); Native.axpb(Ctx.get, handle, b, 0.0, out); new SubMatrix(out, rows, cols)
  }

  /** Matrix x vector (was Breeze `BDM * BDV` -> dgemv): a vector is a block with one column. */
  def multiply(v: SubMatrix): SubMatrix = {
    require(v.cols == 1, s"expected a column vector, got ${v.rows} x ${v.cols}")
    if (isSparse) throw new IllegalArgumentException(s"Not supported multiply-operator between matrices sparsity " +
      s"with $isSparse and vector: class edu.nju.pasalab.marlin.matrix.DenseVector")
    val y = fresh(rows, 1); Native.gemv(Ctx.get, handle, v.handle, y, false); new SubMatrix(y, rows, 1)
  }

  /** `denseBlock.t.copy` of BlockMatrix.transpose (matrix/BlockMatrix.scala:514-523). */
  private[marlin] def transposeCopy(): SubMatrix = {
    val out = fresh(cols, rows); Native.transpose(Ctx.get, handle, out); new SubMatrix(out, cols, rows)
  }

  private[marlin] def sum(): Double = Native.sum(Ctx.get, handle)

  /** Breeze `.copy`: a packed device copy (the in-place factorizations work on one). */
  private[marlin] def copy(): SubMatrix = {
    val out = fresh(rows, cols); Native.copy(Ctx.get, handle, out); new SubMatrix(out, rows, cols)
  }

  private[marlin] def release(): Unit =
    if (isSparse) Native.sparseFree(Ctx.get, sparseHandle) else Native.free(Ctx.get, handle)

  override protected def finalize(): Unit = release()
}

private[marlin] object SubMatrix {
  def uploadSparse(m: SparseMatrix): Long = {
    val cols = m.values.map(v => if (v == null) (Array.empty[Int], Array.empty[Double]) else (v.indices.get, v.values.get))
    val colptr = cols.scanLeft(0)(_ + _._1.length)
    Native.sparseUpload(Ctx.get, m.numRows, m.numCols, colptr, cols.flatMap(_._1), cols.flatMap(_._2))
  }
}

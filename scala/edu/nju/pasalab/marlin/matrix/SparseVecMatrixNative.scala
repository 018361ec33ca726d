package edu.nju.pasalab.marlin.matrix

import breeze.linalg.{SparseVector => BSV}

/**
 * The product of `SparseVecMatrix.multiplySparse` (matrix/SparseVecMatrix.scala:22-50) for one partition of A's rows on the
 * GPU: the partition's rows and the whole of B (collected or broadcast by the caller) are flattened to CSR, one native call
 * (`Native.spvecMultiply` -> `mb_spvec_multiply_host`) multiplies them row by row in float32, and the entries come back as
 * ((row id, column), value), the element type of the reference's `CoordinateMatrix`.  Every entry sums its float32
 * products in the row's stored order (k ascending) from the first one, so the result does not depend on the partitioning.
 * Deviations (DESIGN 3.11): the order is fixed where Spark's shuffle order is not; this.nCols != other.nRows and repeated
 * or unsorted ids are errors.
 *
 * NOT compiled in the marlin_b200 repository (its image has no JVM).
 */
private[marlin] object SparseVecMatrixNative {
  /** One partition of A's rows times B (bRows: B's rows, ids in [0, bNumRows)). */
  def multiplyPartition(aRows: Array[(Long, BSV[Double])], aNumCols: Long, bRows: Array[(Long, BSV[Double])], bNumRows: Long,
                        bNumCols: Long): Array[((Long, Long), Float)] = {
    require(aNumCols == bNumRows, s"multiplySparse: this.nCols $aNumCols does not match other.nRows $bNumRows")
    require(bNumRows <= Int.MaxValue && bNumCols <= Int.MaxValue, "multiplySparse: dimensions above 2^31 - 1")
    val (aRowptr, aColidx, aValues) = flatten(aRows.map(_._2))
    val byId = new Array[BSV[Double]](bNumRows.toInt)             // B over ids [0, nRows), absent ids empty
    for ((id, v) <- bRows) {
      require(id >= 0 && id < bNumRows && byId(id.toInt) == null, s"SparseVecMatrix: bad or repeated row id $id")
      byId(id.toInt) = v
    }
    val (bRowptr, bColidx, bValues) = flatten(byId.map(v => if (v == null) BSV.zeros[Double](bNumCols.toInt) else v))
    val ctx = Ctx.get
    val c = Native.spvecMultiply(ctx, aRows.length, bNumRows.toInt, aRowptr, aColidx, aValues, bNumCols.toInt, bRowptr,
      bColidx, bValues)
    try {
      val nnz = Native.sparseNnz(c).toInt
      val rows = new Array[Int](nnz)
      val cols = new Array[Int](nnz)
      val vals = new Array[Float](nnz)
      Native.spvecCoo(ctx, c, rows, cols, vals)
      Array.tabulate(nnz)(q => ((aRows(rows(q))._1, cols(q).toLong), vals(q)))
    } finally Native.sparseFree(ctx, c)
  }

  /** Row pointers, column indices and values of rows given as BSVs, each in its active (stored) order. */
  private def flatten(rows: Array[BSV[Double]]): (Array[Int], Array[Int], Array[Double]) = {
    val rowptr = new Array[Int](rows.length + 1)
    for (i <- rows.indices) rowptr(i + 1) = rowptr(i) + rows(i).activeSize
    val colidx = new Array[Int](rowptr.last)
    val values = new Array[Double](rowptr.last)
    for (i <- rows.indices) {
      System.arraycopy(rows(i).index, 0, colidx, rowptr(i), rows(i).activeSize)
      System.arraycopy(rows(i).data, 0, values, rowptr(i), rows(i).activeSize)
    }
    (rowptr, colidx, values)
  }
}

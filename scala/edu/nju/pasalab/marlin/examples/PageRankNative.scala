package edu.nju.pasalab.marlin.examples

import breeze.linalg.{DenseVector => BDV}

import edu.nju.pasalab.marlin.matrix.{Ctx, DenseVecMatrix, Native}

/**
 * The loop of examples/PageRank.scala (:41-59) on the GPU: the link rows of `PageRank.loadLinksMatrix` are collected,
 * flattened to sparse rows (the non-zeros of each dense row, targets ascending), and one native call
 * (`Native.pageRank` -> `mb_pagerank_host`) builds the in-links and runs every iteration on the device.  The ranks come
 * back as the example's 2 pieces of ceil(n / 2).  Every rank sums its stored in-links in ascending source order, split at
 * the same block boundary, so the ranks are the dense example's bit for bit (DESIGN 3.12).
 *
 * NOT compiled in the marlin_b200 repository (its image has no JVM).
 */
object PageRankNative {
  def pageRank(linkRows: DenseVecMatrix, iterations: Int): Array[(Int, BDV[Double])] = {
    val n = linkRows.numCols().toInt
    val rows = linkRows.rows.collect().sortBy(_._1)
    val ids = rows.map(_._1)
    val nz = rows.map { case (_, v) => v.toArray.zipWithIndex.filter(_._1 != 0.0) }
    val rowptr = nz.scanLeft(0L)(_ + _.length)
    val targets = nz.flatMap(_.map(_._2))
    val values = nz.flatMap(_.map(_._1))
    val splitLen = math.ceil(n / 2.0).toInt
    val ranks = Array.fill(n)(1.0)
    if (iterations > 0) {
      require(n >= 4, "not supported matrix or vector")
      Native.pageRank(Ctx.get, n, ids, rowptr, targets, values, splitLen.toLong, iterations, ranks)
    }
    Array((0, BDV(ranks.slice(0, splitLen))), (1, BDV(ranks.slice(splitLen, n))))
  }
}

package edu.nju.pasalab.marlin.ml

import scala.collection.mutable.ArrayBuffer

import breeze.linalg.{DenseMatrix => BDM}
import edu.nju.pasalab.marlin.matrix.{Ctx, Native}
import org.apache.spark.broadcast.Broadcast

/**
 * The body of `ALSHelp.updateBlock` (ml/ALSHelp.scala:292-382) on the GPU: the block's normal equations are assembled and
 * solved by one native call (`Native.alsUpdateBlock` -> `mb_als_update_host`).  The messages and the InLinkBlock are
 * flattened in updateBlock's own loop order: product blocks ascending, products ascending within a block, then the
 * ratings of the product's group in order; so every element of every `XtX` and `Xy` is summed in the reference's order.
 * Deviations (DESIGN 3.10): each user has its own `XtX` / `Xy` (the reference shares one per block), the solve is a
 * Cholesky solve, and implicitPrefs needs `YtY` (`computeYtY` of the fixed side on the driver; the reference passes None).
 *
 * NOT compiled in the marlin_b200 repository (its image has no JVM).
 */
private[marlin] object ALSNative {
  def updateBlock(messages: Iterable[(Int, Array[Array[Double]])], inLinkBlock: InLinkBlock, rank: Int, lambda: Double,
                  alpha: Double, implicitPrefs: Boolean, YtY: Option[Broadcast[BDM[Double]]]): Array[Array[Double]] = {
    val blockFactors = messages.toSeq.sortBy(_._1).map(_._2).toArray
    val numUsers = inLinkBlock.elementIds.length
    require(!implicitPrefs || YtY.isDefined, "implicitPrefs needs YtY, the Gramian of the fixed side's factors")
    // the received factor rows back to back, and where each product block starts among them
    val blockStart = blockFactors.scanLeft(0)(_ + _.length)
    val y = new Array[Double](blockStart.last * rank)
    for (b <- blockFactors.indices; p <- blockFactors(b).indices)
      System.arraycopy(blockFactors(b)(p), 0, y, (blockStart(b) + p) * rank, rank)
    // each user's terms in the loop order of :319-357
    val terms = Array.fill(numUsers)(new ArrayBuffer[(Int, Float)])
    for (b <- blockFactors.indices; p <- blockFactors(b).indices) {
      val (us, rs) = inLinkBlock.ratingsForBlock(b)(p)
      var i = 0
      while (i < us.length) { terms(us(i)) += ((blockStart(b) + p, rs(i))); i += 1 }
    }
    val offsets = terms.map(_.length.toLong).scanLeft(0L)(_ + _)
    val partners = terms.flatMap(_.map(_._1))
    val ratings = terms.flatMap(_.map(_._2))
    val yty = YtY.map(_.value.toArray).orNull      // symmetric: either storage order
    val x = new Array[Double](numUsers * rank)
    Native.alsUpdateBlock(Ctx.get, rank, y, inLinkBlock.elementIds.map(_.toLong), offsets, partners, ratings, lambda, alpha,
                          implicitPrefs, yty, x)
    Array.tabulate(numUsers)(u => java.util.Arrays.copyOfRange(x, u * rank, (u + 1) * rank))
  }
}

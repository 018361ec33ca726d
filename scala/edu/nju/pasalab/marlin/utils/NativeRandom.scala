package edu.nju.pasalab.marlin.utils

import edu.nju.pasalab.marlin.matrix.{Ctx, Native, SubMatrix}

/**
 * The input generators of the headline benchmark on the device: what `RandomRDD.getBlockIterator` /
 * `getDenseVecIterator` (rdd/RandomRDD.scala:40-125) do inside `compute` — `generator.setSeed(partition.seed)` followed by
 * `Array.fill(...)(generator.nextValue())` — with the same values, bit for bit, produced in HBM by the XORShift
 * jump-ahead kernel (`mb_fill_uniform`).  The driver-side part is unchanged in meaning: one seed per partition =
 * successive `java.util.Random(seed).nextLong()` (rdd/RandomRDD.scala:28-45), which `Native.partitionSeeds` reproduces so
 * that the driver does not have to construct the RDD partitions to know them.
 */
private[marlin] object NativeRandom {

  /** Block (i, j) of `MTUtils.randomBlockMatrix` (utils/MTUtils.scala:34-61, RandomBlockRDD.compute :184-218): a
   *  blockRows x blockCols block, column-major fill order (BDM.create), U(lo, hi). */
  def uniformBlock(partitionSeed: Long, blockRows: Int, blockCols: Int, lo: Double = 0.0, hi: Double = 1.0): SubMatrix = {
    val blk = Native.alloc(Ctx.get, blockRows, blockCols, Native.F64)
    Native.fillUniform(Ctx.get, blk, partitionSeed, 0L, lo, hi, false)
    new SubMatrix(blk, blockRows, blockCols)
  }

  /** The `size` rows of one partition of `MTUtils.randomDenVecMatrix` (utils/MTUtils.scala:63-75, RandomDenVecRDD): the
   *  rows are generated one after the other from the partition's stream, so the shard is ONE row-major fill of
   *  size x vectorSize values; returned as a device block holding the shard's rows back to back. */
  def uniformRows(partitionSeed: Long, size: Int, vectorSize: Int, lo: Double = 0.0, hi: Double = 1.0): SubMatrix = {
    val blk = Native.alloc(Ctx.get, vectorSize, size, Native.F64)          // column j of the block = row j of the shard
    Native.fillUniform(Ctx.get, blk, partitionSeed, 0L, lo, hi, false)
    new SubMatrix(blk, vectorSize, size).t                             // seen as size x vectorSize, no copy
  }

  /** `uniformBlock` with `StandardNormalGenerator(mean, variance)` (utils/RandomDataGenerator.scala:70-82): the block's
   *  values are mean + sqrt(variance) * nextGaussian() of its partition stream, bit for bit (`mb_fill_normal`). */
  def normalBlock(partitionSeed: Long, blockRows: Int, blockCols: Int, mean: Double = 0.0, variance: Double = 1.0): SubMatrix = {
    val blk = Native.alloc(Ctx.get, blockRows, blockCols, Native.F64)
    Native.fillNormal(Ctx.get, blk, partitionSeed, mean, variance, false)
    new SubMatrix(blk, blockRows, blockCols)
  }

  /** `uniformRows` with `StandardNormalGenerator(mean, variance)`: one stream across the partition's rows, so a pair of
   *  Gaussians may straddle two rows, as `Array.fill` in `RandomDenVecRDD.compute` draws them. */
  def normalRows(partitionSeed: Long, size: Int, vectorSize: Int, mean: Double = 0.0, variance: Double = 1.0): SubMatrix = {
    val blk = Native.alloc(Ctx.get, vectorSize, size, Native.F64)          // column j of the block = row j of the shard
    Native.fillNormal(Ctx.get, blk, partitionSeed, mean, variance, false)
    new SubMatrix(blk, vectorSize, size).t                             // seen as size x vectorSize, no copy
  }

  /** A sparse block of `MTUtils.randomBlockMatrix(..., sparseInfo = (true, density))` (RandomRDD.scala:97-99,
   *  SparseMatrix.rand, Matrices.scala:157-173), seeded: s = (blockCols * density).toInt rows per column (density <= 0
   *  and s > blockRows are IllegalArgumentException), values from the block's partition stream, rows by selection
   *  sampling (mb_fill_sparse_uniform). */
  def sparseBlock(partitionSeed: Long, blockRows: Int, blockCols: Int, density: Double): SubMatrix = {
    val s = Native.sparseColumnCount(blockRows, blockCols, density)
    val sp = Native.sparseAlloc(Ctx.get, blockRows, blockCols, s.toLong * blockCols)
    Native.fillSparseUniform(Ctx.get, sp, partitionSeed)
    new SubMatrix(0L, blockRows, blockCols, sp)
  }

  /** Seeds of the `numPartitions` partitions of a RandomRDD built with `seed` (rdd/RandomRDD.scala:28-45). */
  def partitionSeeds(seed: Long, numPartitions: Int): Array[Long] = Native.partitionSeeds(seed, numPartitions)

  /** Block extents of `RandomBlockRDD.compute` (:199-211): every block is ceil(total / parts) long except the last one of
   *  its direction, which takes what is left when the regular length overshoots. */
  def blockExtent(total: Long, parts: Int, index: Int): Int = {
    val regular = Native.blockLen(total, parts)(0)                         // ceil(total / parts)
    if (index == parts - 1 && regular.toLong * parts > total) (total - regular.toLong * (parts - 1)).toInt else regular
  }
}

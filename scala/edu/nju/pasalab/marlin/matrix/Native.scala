package edu.nju.pasalab.marlin.matrix

/**
 * JNI surface of libmarlin_b200.so (C ABI: include/marlin_b200.h; veneer: jni/marlin_b200_jni.c).
 * One `@native` per exported entry the Scala side needs; handles (contexts, blocks, communicators) travel as `Long`.
 * A non-zero status comes back as IllegalArgumentException (bad argument / dimension mismatch / unsupported grid —
 * the cases the reference guards with `require`) or RuntimeException (CUDA failure, empty collection, peer timeout).
 *
 * NOT compiled in the marlin_b200 repository (its image has no JVM); tests/test_jni_veneer.py checks that every
 * `@native` below has its `Java_edu_nju_pasalab_marlin_matrix_Native_00024_*` twin in the C file.
 */
object Native {
  System.loadLibrary("marlin_b200_jni") // links libmarlin_b200.so

  val F64 = 0; val BF16 = 1; val F32 = 2

  // lifetime (one context per executor thread or per executor: see Ctx)
  @native def init(device: Int): Long
  @native def shutdown(ctx: Long): Unit
  @native def synchronize(ctx: Long): Unit
  @native def version(): String

  // blocks: a Breeze DenseMatrix record (data, offset, rows, cols, majorStride, isTranspose) moved to HBM
  @native def upload(ctx: Long, data: Array[Double], offset: Int, rows: Int, cols: Int, majorStride: Int,
                     isTranspose: Boolean, storeAs: Int): Long
  @native def download(ctx: Long, blk: Long, out: Array[Double], ld: Int): Unit
  @native def alloc(ctx: Long, rows: Int, cols: Int, dtype: Int): Long
  @native def free(ctx: Long, blk: Long): Unit
  @native def viewT(ctx: Long, blk: Long): Long
  @native def slice(ctx: Long, blk: Long, r0: Int, r1: Int, c0: Int, c1: Int): Long

  // per-block kernels
  @native def gemm(ctx: Long, a: Long, b: Long, c: Long, accumulate: Boolean): Unit
  @native def add(ctx: Long, a: Long, b: Long, out: Long): Unit
  @native def sub(ctx: Long, a: Long, b: Long, out: Long): Unit
  @native def hadamard(ctx: Long, a: Long, b: Long, out: Long): Unit
  @native def axpb(ctx: Long, a: Long, alpha: Double, beta: Double, out: Long): Unit
  @native def div(ctx: Long, a: Long, b: Double, bOverA: Boolean, out: Long): Unit
  @native def transpose(ctx: Long, a: Long, out: Long): Unit
  @native def copy(ctx: Long, a: Long, out: Long): Unit
  @native def sum(ctx: Long, a: Long): Double
  @native def gemv(ctx: Long, a: Long, x: Long, y: Long, accumulate: Boolean): Unit
  @native def dot(ctx: Long, x: Long, y: Long): Double
  @native def ger(ctx: Long, x: Long, y: Long, out: Long): Unit
  @native def fillUniform(ctx: Long, blk: Long, partitionSeed: Long, first: Long, lo: Double, hi: Double,
                          rowMajor: Boolean): Unit
  @native def setFp64Mode(ctx: Long, mode: Int, slices: Int): Unit

  // the Breeze/LAPACK leaves of luDecompose / choleskyDecompose / inverse (brzLU, brzCholesky, brzInv, `\`)
  @native def lu(ctx: Long, a: Long, permOut: Array[Int]): Unit
  @native def cholesky(ctx: Long, a: Long): Unit
  @native def inverse(ctx: Long, a: Long, out: Long): Unit
  // the local steps of computeSVD: Gramian, symmetric eigendecomposition (returns the sweep count), mode chooser, rank
  @native def gramian(ctx: Long, a: Long, g: Long): Unit
  @native def syev(ctx: Long, g: Long, v: Long, wOut: Array[Double]): Int
  @native def svdMode(n: Long, k: Int, mode: String): Int // 0 local-svd, 1 local-eigs, 2 dist-eigs
  @native def svdRank(sigmas: Array[Double], k: Int, rCond: Double): Int
  @native def trsm(ctx: Long, t: Long, lower: Boolean, unitDiagonal: Boolean, b: Long): Unit

  // whole multiplies on one GPU
  @native def matmulBlocked(ctx: Long, aTiles: Array[Long], bTiles: Array[Long], m: Int, k: Int, n: Int,
                            cTiles: Array[Long]): Unit
  @native def matmulRowsharded(ctx: Long, aRows: Long, b: Long, cRows: Long): Unit
  @native def matmulRowshardedHost(ctx: Long, aRows: Array[Double], rows: Long, k: Int, b: Array[Double], n: Int,
                                   cRows: Array[Double]): Unit
  @native def dgemmHost(ctx: Long, transA: Boolean, transB: Boolean, m: Int, n: Int, k: Int, alpha: Double,
                        a: Array[Double], aOff: Int, lda: Int, b: Array[Double], bOff: Int, ldb: Int, beta: Double,
                        c: Array[Double], cOff: Int, ldc: Int): Unit

  // BlockMatrix.multiply across the GPUs of one box
  @native def commInit(ctx: Long, rank: Int, world: Int, session: String): Long
  @native def commDestroy(comm: Long): Unit
  @native def commBarrier(comm: Long): Unit
  @native def commCheck(comm: Long): Unit
  @native def commAbort(comm: Long): Unit
  @native def distPlan(m: Int, k: Int, n: Int, world: Int): Array[Int] // m*k*n product ranks, then m*n C owners
  @native def matmulBlockedDist(comm: Long, aTiles: Array[Long], aOwner: Array[Int], bTiles: Array[Long],
                                bOwner: Array[Int], m: Int, k: Int, n: Int, rowLen: Array[Int], kLen: Array[Int],
                                colLen: Array[Int], dtype: Int, cTiles: Array[Long]): Unit

  // driver-side integer logic, bit-identical to the Scala it stands in for
  @native def chooseSplit(m: Long, k: Long, n: Long, cores: Int): Array[Int]
  @native def chooseStrategy(aRows: Long, aCols: Long, bCols: Long, cores: Int, thresholdMb: Int,
                             otherIsBlock: Boolean): Array[Int] // strategy, m, k, n
  @native def multPartition(i: Int, j: Int, kk: Int, m: Int, k: Int, n: Int): Int
  @native def elemPartition(row: Int, col: Int, blksByCol: Int): Int
  @native def blockLen(total: Long, parts: Int): Array[Int]
  @native def hashSeed(seed: Long): Long
  @native def partitionSeeds(seed: Long, numPartitions: Int): Array[Long]
}

/**
 * The executor-side context: one `mb_ctx` per task thread (Spark `local[N]` runs N task threads in one JVM —
 * LocalSparkContext.scala:11 — and a context owns one stream plus scratch), on the GPU this executor was given
 * (`marlin.b200.device`, default 0; with one executor process per GPU, CUDA_VISIBLE_DEVICES makes that device 0).
 */
object Ctx {
  private val device = sys.props.getOrElse("marlin.b200.device", "0").toInt
  private val local = new ThreadLocal[java.lang.Long] {
    override def initialValue(): java.lang.Long = Native.init(device)
  }
  def get: Long = local.get()
}

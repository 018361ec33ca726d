/*
 * marlin_b200.h — C ABI of libmarlin_b200.so, the H100 (sm_90a) drop-in for the dense
 * block-matrix hot path of PasaLab/marlin (edu.nju.pasalab.marlin.matrix).
 *
 * The reference has no FFI of its own; its only native seam is Breeze -> netlib-java
 * BLAS.dgemm (third-party, not in the tree).  The entry points below are what a JNI veneer
 * for edu.nju.pasalab.marlin.matrix.{SubMatrix,BlockMatrix,DenseVecMatrix} and
 * edu.nju.pasalab.marlin.utils.MTUtils would bind (see INTEGRATION.md for the Scala/JNI side).
 * Every entry cites the reference code it replaces (paths relative to the reference's
 * src/main/scala/edu/nju/pasalab/marlin/).
 *
 * Conventions
 *   - plain C, no torch / C++ types; all functions return int32 status (0 = MB_OK, <0 = error);
 *     mb_last_error() returns a thread-local message for the last failing call.  An entry that returns a
 *     new block or sparse handle through *out sets *out to NULL on failure and leaves nothing allocated.
 *   - one mb_ctx per process and GPU (one process per GPU, like one Spark executor per device).
 *   - a block (mb_block) is the device-resident analogue of SubMatrix.denseBlock: Breeze
 *     DenseMatrix semantics (data, offset, rows, cols, majorStride, isTranspose), column-major:
 *        element(r,c) = data[offset + r + c*ld]            if !is_transpose
 *                     = data[offset + c + r*ld]            if  is_transpose
 *   - there is NO CPU fallback: without a CUDA device every compute entry returns MB_ERR_CUDA.
 */
#ifndef MARLIN_B200_H
#define MARLIN_B200_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default)   /* the library is built with -fvisibility=hidden */
#endif

#define MB_OK                 0
#define MB_ERR_INVALID_ARG   -1   /* -> IllegalArgumentException on the JVM side            */
#define MB_ERR_DIM_MISMATCH  -2   /* -> IllegalArgumentException ("Dimension mismatch ...")  */
#define MB_ERR_UNSUPPORTED   -3   /* -> IllegalArgumentException ("currently not supported") */
#define MB_ERR_CUDA          -4   /* -> RuntimeException                                     */
#define MB_ERR_OOM           -5
#define MB_ERR_EMPTY         -6   /* -> RuntimeException (empty RDD: DistributedMatrixSuite "empty rows") */
#define MB_ERR_IO            -9   /* a file that cannot be opened or written -> java.io.IOException */

typedef enum { MB_F64 = 0, MB_BF16 = 1, MB_F32 = 2 } mb_dtype;

typedef struct mb_ctx   mb_ctx;
typedef struct mb_block mb_block;
typedef struct mb_sparse mb_sparse;

/* ---- lifetime (SparkContext lifetime in the reference) --------------------------------- */
int32_t     mb_init(int32_t device, mb_ctx** out);
int32_t     mb_shutdown(mb_ctx* ctx);
const char* mb_last_error(void);
const char* mb_version(void);
/* Use an externally owned stream (e.g. torch's current stream) for every later call.  The handle is
 * used as CUDA would: NULL is the legacy default stream.  mb_reset_stream returns to the ctx's own
 * (non-blocking) stream, which is what a fresh ctx uses. */
int32_t     mb_set_stream(mb_ctx* ctx, void* cuda_stream);
int32_t     mb_reset_stream(mb_ctx* ctx);
int32_t     mb_synchronize(mb_ctx* ctx);
/* Number of kernels enqueued by calls on ctx since init, the kernel nodes of graph launches included (bench.py's
 * gpu_launches).  Memsets, copies and stream memory operations are not counted; a call that launches nothing adds nothing. */
int64_t     mb_launch_count(mb_ctx* ctx);
/* CUDA-event timing on the ctx stream, so callers can time kernels on the launching stream. */
int32_t     mb_timer_start(mb_ctx* ctx);
int32_t     mb_timer_stop(mb_ctx* ctx, float* ms_out);

/* ---- blocks: `new SubMatrix(denseMatrix = ...)` (matrix/SubMatrix.scala:16-20) ---------- */
int32_t mb_block_alloc(mb_ctx* ctx, int32_t rows, int32_t cols, mb_dtype dtype, mb_block** out);
/* Non-owning view over device memory someone else allocated (torch tensor, NCCL buffer). */
int32_t mb_block_wrap(mb_ctx* ctx, void* device_ptr, int64_t offset, int32_t rows, int32_t cols,
                      int32_t ld, int32_t is_transpose, mb_dtype dtype, mb_block** out);
/* Host fp64 (Breeze data/offset/majorStride/isTranspose) -> packed device block (ld = rows),
 * optionally rounded to bf16 (round-to-nearest-even) for the bf16 path. */
int32_t mb_block_upload(mb_ctx* ctx, const double* host, int64_t offset, int32_t rows, int32_t cols,
                        int32_t ld, int32_t is_transpose, mb_dtype store_as, mb_block** out);
/* toBreeze()/collect (matrix/BlockMatrix.scala:70-85): packed column-major fp64, leading dim ld. */
int32_t mb_block_download(mb_ctx* ctx, const mb_block* blk, double* host, int32_t ld);
int32_t mb_block_free(mb_ctx* ctx, mb_block* blk);
int32_t mb_block_info(const mb_block* blk, int32_t* rows, int32_t* cols, int32_t* ld,
                      int32_t* is_transpose, int32_t* dtype, void** device_ptr);
/* Optional: a cudaEvent_t that completes when the block's contents are final (blocks are immutable values, like the
 * blocks of a cached RDD).  mb_matmul_blocked_dist then offers such tiles to the other ranks as soon as that event has
 * completed instead of after everything queued on the ctx stream — the pulls of multiply s+1 overlap the products of
 * multiply s.  The event must outlive the calls that use the block; NULL (default) = ordered on the ctx stream. */
int32_t mb_block_set_ready_event(mb_block* blk, void* cuda_event);
/* Breeze `.t` (no copy) and `m(r0 until r1, c0 until c1)` (a view, majorStride = parent rows),
 * as used by BlockMatrix.scala:198,213,299. */
int32_t mb_block_view_t(mb_ctx* ctx, const mb_block* blk, mb_block** out);
int32_t mb_block_slice(mb_ctx* ctx, const mb_block* blk, int32_t r0, int32_t r1, int32_t c0, int32_t c1,
                       mb_block** out);

/* ---- a1: SubMatrix.multiply (matrix/SubMatrix.scala:87-91, :107-111; inline twins
 *      matrix/DenseVecMatrix.scala:122,129,1676) -> Breeze `*` -> netlib dgemm -------------- */
/* C = A*B (accumulate=0) or C += A*B (accumulate=1; the k-way reduceByKey sum of
 * BlockMatrix.scala:177 fused into the product).  fp64: DMMA tensor-core kernel (TMA staged).
 * bf16 inputs: wgmma kernel with fp32 register accumulation, C may be F32 or BF16; any shape, offset and ld
 * (operands the TMA cannot address are copied to a packed buffer first), K = 0 gives C = 0, and an F32 C is built
 * from accumulation chains of at most MARLIN_B200_BF16_KCHAIN (default 8192) k per launch. */
int32_t mb_block_gemm(mb_ctx* ctx, const mb_block* A, const mb_block* B, mb_block* C, int32_t accumulate);
/* The trailing (Schur) update of the dist-mode block factorizations, as one call for a rank's whole step:
 * C[e] = C[e] - A[e]*B[e] for e < count, in place, fp64.  It replaces the per-block `multiply` + `subtract` of
 * matrix/DenseVecMatrix.scala:421-427 (LU), :531-549 (Cholesky, B[e] a transposed view) and :666-671 (inverse).
 * Each C[e] is bit for bit mb_block_gemm(A[e], B[e]) -> tmp followed by mb_block_sub(C[e], tmp), with or without
 * mb_set_dmma_reference.  Entries the DMMA GEMM would run are packed, in order, into grouped launches of at most
 * 64 entries and 32 distinct A and 32 distinct B operands each (a transposed B is copied once to column-major
 * first); the others run as exactly those two calls.  MB_ERR_DIM_MISMATCH when an entry's shapes disagree,
 * MB_ERR_INVALID_ARG when an output overlaps another output or any operand; count == 0 launches nothing. */
int32_t mb_block_schur_update(mb_ctx* ctx, int32_t count, mb_block* const* C, const mb_block* const* A,
                              const mb_block* const* B);
/* Same GEMM on raw device pointers (column-major, BLAS trans flags 'N'/'T'). */
int32_t mb_dgemm_device(mb_ctx* ctx, char transa, char transb, int32_t m, int32_t n, int32_t k,
                        double alpha, const double* A, int32_t lda, const double* B, int32_t ldb,
                        double beta, double* C, int32_t ldc);
/* The third-party seam itself: com.github.fommil.netlib.BLAS.dgemm(transa, transb, m, n, k, alpha,
 * a, aOffset, lda, b, bOffset, ldb, beta, c, cOffset, ldc) with HOST arrays (JVM double[]).
 * Uploads, multiplies on the GPU, downloads C.  This is the end-to-end (e2e) entry bench.py times. */
int32_t mb_dgemm_host(mb_ctx* ctx, char transa, char transb, int32_t m, int32_t n, int32_t k,
                      double alpha, const double* a, int64_t a_offset, int32_t lda,
                      const double* b, int64_t b_offset, int32_t ldb,
                      double beta, double* c, int64_t c_offset, int32_t ldc);
/* fp64 arithmetic mode of the block GEMM.  MB_FP64_NATIVE (default): the DMMA kernel, true IEEE fp64 FMAs.
 * MB_FP64_INT8_SPLIT: large 'N','N' products run on the int8 tensor cores (wgmma .s32.s8.s8) from `slices`
 * 7-bit digit planes per operand (Ozaki split; 2..8, 7 recommended): error <= ~K * 2^(-7*slices+2) relative to
 * rowmax(A) * colmax(B), i.e. well inside 1e-10 for well-scaled data but NOT an element-wise fp64 guarantee, hence
 * opt-in.  Products the split does not cover (transposed views, small blocks, K too large for exact int32
 * accumulation) silently use the native kernel.  Rows of A / columns of B holding a NaN or Inf are left out of the split
 * and their entries of C recomputed in plain fp64, so NaN / Inf propagate as with the native kernel. */
#define MB_FP64_NATIVE      0
#define MB_FP64_INT8_SPLIT  1   /* 7-bit digits (|d| <= 64):  P = 7*slices - 1 fractional bits, K*slices < 2^19  */
#define MB_FP64_INT8_SPLIT8 2   /* 8-bit digits (|d| <= 128): P = 8*slices - 2 fractional bits, K*slices < 2^17;
                                   slices = 5 gives 38 bits in 15 int8 GEMMs (vs 42 bits in 21 for 7-bit x 6)     */
int32_t mb_set_fp64_mode(mb_ctx* ctx, int32_t mode, int32_t slices);

/* Force the generic (non-TMA, CUDA-core DFMA) kernel: test hook + path for odd ld / unaligned views. */
int32_t mb_dgemm_device_generic(mb_ctx* ctx, char transa, char transb, int32_t m, int32_t n, int32_t k,
                                double alpha, const double* A, int32_t lda, const double* B, int32_t ldb,
                                double beta, double* C, int32_t ldc);

/* Test and measurement hook, not a user option (off by default).  on != 0: every fp64 DMMA kernel that later calls on ctx
 * launch (block and device GEMMs, the grouped blocked multiply, the distributed multiply, the row-sharded multiply, the
 * factorizations' updates and the Gramian) runs its m8n8k4 instance (SASS DMMA.8x8x4) instead of the m16n8k4 one
 * (DMMA.16x8x4, twice the issue rate on H100).  The two share all source but the instruction shape and give the same
 * results bit for bit: the m8n8k4 instances are the reference the m16n8k4 kernels are tested against and the A/B switch
 * for measuring them. */
int32_t mb_set_dmma_reference(mb_ctx* ctx, int32_t on);

/* ---- a2/a10: SubMatrix.add/subtract/scalar ops (matrix/SubMatrix.scala:41-85,123-131),
 *      BlockMatrix.subtractBy/divideBy (matrix/BlockMatrix.scala:414-452) ------------------- */
int32_t mb_block_add(mb_ctx* ctx, const mb_block* A, const mb_block* B, mb_block* out);      /* A + B */
int32_t mb_block_sub(mb_ctx* ctx, const mb_block* A, const mb_block* B, mb_block* out);      /* A - B */
int32_t mb_block_hadamard(mb_ctx* ctx, const mb_block* A, const mb_block* B, mb_block* out); /* A :* B (BlockMatrix.scala:494-500) */
/* out = alpha*A + beta  (add(b): alpha=1; multiply(b): beta=0; subtractBy(b): alpha=-1, beta=b) */
int32_t mb_block_axpb(mb_ctx* ctx, const mb_block* A, double alpha, double beta, mb_block* out);
/* BDM.zeros / BDM.fill: every element of the (possibly strided) block := value */
int32_t mb_block_fill(mb_ctx* ctx, mb_block* blk, double value);
/* out = A / b  (true IEEE division, SubMatrix.divide) and out = b / A (divideBy) */
int32_t mb_block_div(mb_ctx* ctx, const mb_block* A, double b, int32_t b_over_a, mb_block* out);
/* ---- a9: BlockMatrix.transpose -> denseBlock.t.copy (matrix/BlockMatrix.scala:514-523) -- */
int32_t mb_block_transpose(mb_ctx* ctx, const mb_block* A, mb_block* out);
/* Materialise a (possibly strided / transposed) view into a packed block (Breeze `.copy`). */
int32_t mb_block_copy(mb_ctx* ctx, const mb_block* A, mb_block* out);
/* BlockMatrix.sum per block (matrix/BlockMatrix.scala:467-472) */
int32_t mb_block_sum(mb_ctx* ctx, const mb_block* A, double* sum_out);

/* ---- DenseVecMatrix.norm(mode) (matrix/DenseVecMatrix.scala:975-999) on one row shard.  The reference's "1" never sums
 *      (its per-row map is lazy and discarded) and its "inf" sums signed values; these are the norms its comment names:
 *      the largest column sum of |a|, the largest row sum of |a|, and sqrt(sum a^2) (a TODO there).  "2" stays
 *      unsupported. ---- */
#define MB_NORM_ONE 0
#define MB_NORM_INF 1
#define MB_NORM_FRO 2
/* The mode string of norm(mode): "1", "inf" or "fro" -> MB_NORM_ONE / MB_NORM_INF / MB_NORM_FRO in *kind; anything else
 * (also "2") is MB_ERR_INVALID_ARG "Do not support mode <mode>.".  Pure logic, no GPU needed. */
int32_t mb_norm_mode(const char* mode, int32_t* kind);
/* One pass over any fp64 view A (m x n, element strides as the block says; a row shard's transposed view is read in
 * place).  Blocking.  Every result is the same bits on every run.
 *   MB_NORM_ONE: col_sums (an fp64 vector of n elements: one row or one column) := the column sums of |a|, each the sum of
 *                fixed chunks of rows, a chunk summed in row order, the chunk partials in chunk order; *out (may be NULL)
 *                := the largest of them.
 *   MB_NORM_INF: *out := the largest row sum of |a|, each row a left fold s = s + |a_rc| in column order from 0.0.
 *   MB_NORM_FRO: out[0..2] := the small, medium and big accumulators of sum a^2 as LAPACK 3.10 dnrm2 (Blue's algorithm)
 *                keeps them; mb_norm_fro turns them into the norm.  col_sums is not used by INF and FRO.
 * "Largest" is java.lang.Double.compare's order (RDD.max()): a NaN anywhere is the result.  A view with no rows, or the
 * 1-norm of no columns, is MB_ERR_EMPTY "empty collection". */
int32_t mb_block_norm(mb_ctx* ctx, const mb_block* A, int32_t kind, mb_block* col_sums, double* out);
/* The Frobenius norm of `count` shards from their accumulator triples acc[3 * i .. 3 * i + 2] (mb_block_norm,
 * MB_NORM_FRO), added in index order, then dnrm2's final combination: no spurious overflow or underflow.  Pure logic. */
int32_t mb_norm_fro(const double* acc, int32_t count, double* out);

/* ---- vector side of the path (SURVEY 8f-4): a vector is a block with one column (or one row) ----
 * y = A x (+ y): SubMatrix.multiply(v: Vector) (matrix/SubMatrix.scala:131-139) -> Breeze `BDM * BDV` -> netlib dgemv;
 * used per block by BlockMatrix.multiply(v: DistributedVector / BDV) (matrix/BlockMatrix.scala:240-274), whose
 * reduceByKey sum is `accumulate`.  A may be a transposed view (row-major rows of a DenseVecMatrix,
 * matrix/DenseVecMatrix.scala:178-191).  Reads A once: 8*rows*cols bytes. */
int32_t mb_block_gemv(mb_ctx* ctx, const mb_block* A, const mb_block* x, mb_block* y, int32_t accumulate);
/* x^T y: DistributedVector.multiply, row x column case (matrix/DistributedVector.scala:164-176) -> Breeze `v.t * w`. */
int32_t mb_block_dot(mb_ctx* ctx, const mb_block* x, const mb_block* y, double* dot_out);
/* out = x y^T: DistributedVector.multiply, column x row case (matrix/DistributedVector.scala:149-161)
 * -> Breeze `v * w.t` -> dgemm with k = 1. */
int32_t mb_block_ger(mb_ctx* ctx, const mb_block* x, const mb_block* y, mb_block* out);

/* ---- f4: the local step of DenseVecMatrix.luDecompose / choleskyDecompose / inverse
 *      (matrix/DenseVecMatrix.scala:283-466, 475-561, 568-764), which the reference hands to Breeze -> LAPACK
 *      (brzLU = dgetrf, brzCholesky = dpotrf, brzInv = dgetrf + dgetri, `\` = triangular / general solves).
 *      Recursive on the device: the flops run in the DMMA GEMM, the leaves in small panel kernels. ---- */
/* In place: unit-lower L and U packed like dgetrf; perm_out (rows entries, host, may be NULL) receives the reference's
 * permutation array: row i of L*U is row perm_out[i] of A.  A singular pivot is not an error (as with brzLU). */
int32_t mb_block_lu(mb_ctx* ctx, mb_block* A, int32_t* perm_out);
/* In place: L (lower, A = L L^T), strict upper triangle zeroed (Breeze `cholesky`); reads the lower triangle only.
 * MB_ERR_CUDA ("not positive definite") if a pivot is not positive. */
int32_t mb_block_cholesky(mb_ctx* ctx, mb_block* A);
/* out = A^-1 (partial-pivoting LU + two triangular solves of the permuted identity); MB_ERR_CUDA if exactly singular. */
int32_t mb_block_inverse(mb_ctx* ctx, const mb_block* A, mb_block* out);
/* T X = B in place (B := X), T triangular (lower / upper, unit or explicit diagonal); with transposed views of T and B
 * this also covers X T = B.  Used for `l \ b` and `b * inv(u)` of the block algorithms. */
int32_t mb_block_trsm(mb_ctx* ctx, const mb_block* T, int32_t lower, int32_t unit_diagonal, mb_block* B);

/* ---- f5: DenseVecMatrix.computeSVD (matrix/DenseVecMatrix.scala:1531-1652): the Gramian A^T A, its symmetric
 *      eigendecomposition and the two decisions of the reference's driver code.  U = A (V_k S_k^-1) is then
 *      mb_block_div on column views of V and mb_matmul_rowsharded. ---- */
#define MB_ERR_NO_CONVERGENCE -8   /* the eigensolver hit its sweep cap -> IllegalStateException (:1798-1807)      */
/* DenseVecMatrix.computeGramianMatrix (:1464-1486, dspr + triuToFull): G (n x n) = A^T A for any fp64 view A (m x n),
 * e.g. the transposed view of a row shard.  Exactly symmetric; bitwise reproducible from run to run (fixed-order split-K
 * sum).  More than 65535 columns is MB_ERR_INVALID_ARG, as in the reference. */
int32_t mb_block_gramian(mb_ctx* ctx, const mb_block* A, mb_block* G);
/* Bytes of temporary device memory mb_block_gramian takes for an m x n operand on num_sms SMs (TMA-addressable operand;
 * other views take none): the split-K partials, 0 unless the lower triangle has fewer than two waves of 128 x 128 tiles,
 * never more than 256 MiB.  Stream-ordered (cudaMallocAsync), returned when the call's work completes.  Pure logic. */
int64_t mb_gramian_workspace_bytes(int64_t n, int64_t m, int32_t num_sms);
/* brzSvd(G) / EigenValueDecomposition.symmetricEigs (:1596-1606, :1725-1834) for a symmetric G (lower triangle read):
 * all n eigenvalues into the HOST array w_out, ordered by |w| descending (ties: lower index first) — what dgesdd returns
 * as singular values of a symmetric G — and the matching orthonormal eigenvectors as the columns of V (n x n).
 * sweeps_out (may be NULL) receives the number of Jacobi sweeps.  Blocking.  Takes 32 * N^2 bytes of temporary device
 * memory (N = n rounded up to even) for the duration of the call.  G is first scaled by the power of two that brings
 * max|g| into [1, 2), so 2^k G gives V and the sweep count of G bit for bit and w * 2^k (while w * 2^k stays normal).
 * A NaN or +-Inf in the lower triangle of G is MB_ERR_INVALID_ARG before any sweep runs (w_out and V unset). */
int32_t mb_block_syev(mb_ctx* ctx, const mb_block* G, mb_block* V, double* w_out, int32_t* sweeps_out);
/* The mode chooser and every `require` of computeSVD (:1565-1604) plus the column cap of computeGramianMatrix
 * (:1466-1468), with the reference's messages.  mode: "auto", "local-svd", "local-eigs" or "dist-eigs"; *compute_mode
 * receives MB_SVD_LOCAL_LAPACK / MB_SVD_LOCAL_ARPACK / MB_SVD_DIST_ARPACK.  Pure integer logic, no GPU needed. */
#define MB_SVD_LOCAL_LAPACK 0
#define MB_SVD_LOCAL_ARPACK 1
#define MB_SVD_DIST_ARPACK  2
int32_t mb_svd_mode(int64_t n, int32_t k, const char* mode, int32_t* compute_mode);
/* The effective rank sk of :1607-1621: the number of leading sigmas >= rcond * sigmas[0], at most min(k, count).
 * Returns sk (>= 0) or a negative error code. */
int32_t mb_svd_rank(const double* sigmas, int32_t count, int32_t k, double rcond);

/* ---- f5, the overload computeSVD(k, computeU, rCond, maxIter, tol, mode) (:1557-1652): the eigs modes run a Lanczos
 *      solver on the device instead of a full decomposition of G.  "dist-eigs" never forms G. ---- */
/* The chooser of that overload: mb_svd_mode's rules and messages, except that the 65535-column cap of
 * computeGramianMatrix applies only to the modes that form G ("local-svd", "local-eigs"); "dist-eigs" takes any n up to
 * INT32_MAX.  max_iter <= 0 is rejected in the eigs modes (ARPACK's info = -4).  Pure logic, no GPU needed. */
int32_t mb_svd_plan(int64_t n, int32_t k, const char* mode, int32_t max_iter, double tol, int32_t* compute_mode);
/* multiplyGramianMatrixBy (:1444-1459) over one shard: y = A^T (A x), or y += it when accumulate != 0.  A is an fp64
 * m x n view; x and y are fp64 vectors of n elements.  A row-major view (a row shard's transposed view, any ld, 8-byte
 * alignment) or a single column is read in place; any other view is first packed into a row-major copy (one more
 * launch and 16 m n more bytes).  Rows n <= 5118 wide cross HBM once (8 m n bytes); wider rows are streamed twice
 * (16 m n).  Fixed summation order, no atomics, every multiply and add rounded separately: the same inputs give the
 * same bits on every run.  m = 0 gives zeros (y unchanged when accumulating).  Two kernel launches when m > 0. */
int32_t mb_block_gram_matvec(mb_ctx* ctx, const mb_block* A, const mb_block* x, mb_block* y, int32_t accumulate);
/* EigenValueDecomposition.symmetricEigs (:1725-1834) by reverse communication, as ARPACK's dsaupd / dseupd loop:
 * thick-restart Lanczos (Wu-Simon; for a symmetric operator equivalent to ARPACK's implicit restart with exact shifts)
 * for the nev eigenvalues of largest magnitude of an n x n symmetric operator, with an ncv-vector basis (the reference
 * uses ncv = min(2 nev, n)).  Each restart keeps nev + min(nconv, (ncv - nev) / 2) Ritz vectors (dsaup2), at most
 * ncv - 1.  A pair is converged when |beta y_last| <= tol max(eps^(2/3), |theta|) (dsconv), or when that residual is
 * already at the operator's rounding level (<= 2^-46 max |theta|); tol <= 0 means eps = 2^-53.  Every new basis
 * vector is orthogonalised against the whole basis by classical Gram-Schmidt run twice.  The start vector is
 * mb_fill_uniform's stream `seed` on [-1, 1), so every rank that uses the same seed starts from the same bits; if the
 * Krylov space becomes invariant a fresh vector from the same stream continues it (dgetv0).  Device memory:
 * 8 n (2 ncv + 3) bytes.  max_iter bounds the restarts; running out is MB_ERR_NO_CONVERGENCE with the reference's
 * info = 1 message. */
typedef struct mb_eigs mb_eigs;
int32_t mb_eigs_create(mb_ctx* ctx, int32_t n, int32_t nev, int32_t ncv, double tol, int32_t max_iter, int64_t seed,
                       mb_eigs** out);
/* One turn of the loop.  *ido == 1: write y = Op x (both device n x 1 views the solver owns) and call again;
 * *ido == 99: done (mb_eigs_result).  At most one host synchronisation per call. */
int32_t mb_eigs_step(mb_ctx* ctx, mb_eigs* eigs, int32_t* ido, mb_block** x, mb_block** y);
/* The nev eigenvalues, descending, into the HOST array w (may be NULL) and their orthonormal eigenvectors into Z (an fp64
 * n x nev block, may be NULL); *nconv and *iters (may be NULL): the converged pairs and the restarts taken.  Blocking. */
int32_t mb_eigs_result(mb_ctx* ctx, mb_eigs* eigs, double* w, mb_block* Z, int32_t* nconv, int32_t* iters);
int32_t mb_eigs_destroy(mb_eigs* eigs);
/* The solver's projected problem on the host: all eigenpairs of a symmetric n x n matrix T (column-major, lower triangle
 * read) by cyclic Jacobi; w receives the eigenvalues descending, Z (column-major n x n) the eigenvectors.  Pure logic. */
int32_t mb_eigs_projected(int32_t n, const double* T, double* w, double* Z);

/* ---- DenseVecMatrix.lr (matrix/DenseVecMatrix.scala:1005-1035): logistic regression by gradient steps over the rows.
 *      `rows` is an fp64 view with one training row per matrix row (a row shard's transposed view is read in place, any
 *      other view is first copied into a row-major buffer).  Column 0 is the label; the features are the row with
 *      column 0 replaced by the intercept 1.  The input is never written.  Per row: margin = -1.0 * (features . w),
 *      sequential in column order with separate multiplies and adds (BLAS ddot as F2J runs it), gradientMul =
 *      1 / (1 + exp(margin)) - label, gradient = features * gradientMul.  The rows' gradients are summed in a fixed
 *      order (bitwise reproducible).  A block with no rows is MB_ERR_EMPTY, a non-fp64 block MB_ERR_UNSUPPORTED. ---- */
/* The sum of the per-row gradients for the weights w: w and grad are HOST arrays of rows->cols doubles.  This is the
 * body of one partition of one iteration.  Blocking. */
int32_t mb_lr_gradient(mb_ctx* ctx, const mb_block* rows, const double* w, double* grad);
/* The whole loop on one device: w = 0, then for i = 1..iters: w = w - delta_i * (step / data_size / sqrt(i)) with
 * delta_i the gradient sum at the current w.  Every iteration is enqueued without a host synchronisation; the final w
 * (rows->cols doubles) goes to the HOST array w_out.  iters <= 0 gives zeros.  data_size is the reference's numRows()
 * (max row id + 1) and must be positive.  Blocking. */
int32_t mb_lr_train(mb_ctx* ctx, const mb_block* rows, int64_t data_size, double step, int32_t iters, double* w_out);

/* ---- CoordinateMatrix.ALS (matrix/CoordinateMatrix.scala:88-98, ml/ALSHelp.scala:34-382).  One side of the problem is the
 *      users (row ids), the other the products (column ids); an entity of a side has a POSITION: block 0's distinct ids
 *      ascending, then block 1's, ... with block = id mod num_blocks (Spark's HashPartitioner).  A side's factors are a
 *      row-major fp64 view (is_transpose = 1, or one column) with one row per position and `rank` columns.
 *      The arithmetic of one entity u is updateBlock's (:292-382), in its order:
 *        A_u = sum of fl(y_i y_j) over u's terms (partner block ascending, partner id ascending, then input order), each
 *              element one sequential sum from 0.0 with separate roundings; implicit: sum of fl(fl(c - 1) fl(y_i y_j)) with
 *              c = fl(1 + fl(alpha |r|));
 *        b_u = sum of fl(r y_i); implicit: sum of fl(c y_i) over the ratings r > 0;
 *        A_u(i, i) += fl(numRatings * lambda), then (implicit) A_u += YtY, the Gramian of the fixed side's factors;
 *        x_u = A_u^-1 b_u by Cholesky (the reference inverts and multiplies: equal within rounding, not bitwise).
 *      A_u never leaves the kernel.  rank < 1 or lambda < 0: MB_ERR_INVALID_ARG; rank > MB_ALS_MAX_RANK: MB_ERR_UNSUPPORTED.
 *      A non-positive pivot (only possible with lambda = 0) is MB_ERR_CUDA "not positive definite" naming the lowest
 *      such entity id. ---- */
#define MB_ALS_MAX_RANK 128
/* Pure host logic (makeOutLinkBlock / makeInLinkBlock, :101-165) for the side whose ids are ent[] (partner[] the other
 * side's ids of the same ratings).  Every id must lie in [0, 2^31 - 1] (MB_ERR_INVALID_ARG otherwise; the reference
 * truncates with toInt).  Writes, with n = the side's distinct ids (returned in *count_out, n <= nnz):
 *   ids_out[n]                 the id of each position
 *   block_offsets_out[nb + 1]  block b holds positions [block_offsets_out[b], block_offsets_out[b + 1])
 *   offsets_out[n + 1]         position p's terms are q in [offsets_out[p], offsets_out[p + 1]), in the order above,
 *   partners_out[nnz], ratings_out[nnz]  the partner's position on the other side and the rating of term q
 *   work_out[n]                positions by rating count descending, ties by position (heaviest first)
 * Duplicated (row, col) entries are kept, each a term of its own, in input order.  Output arrays are sized by nnz. */
int32_t mb_als_links(int64_t nnz, const int64_t* ent, const int64_t* partner, const float* values, int32_t num_blocks,
                     int32_t num_partner_blocks, int64_t* ids_out, int64_t* block_offsets_out, int64_t* offsets_out,
                     int32_t* partners_out, float* ratings_out, int32_t* work_out, int64_t* count_out);
/* Pure host logic (:60-74, randomFactor :170-179): the initial factors of `count` consecutive positions of block `block`
 * of side 0 (users, seed1) or side 1 (products, seed2), row-major into out[count * rank].  seed1 and seed2 are the first
 * two nextInt() of java.util.Random(seed); the block draws from Random(byteswap32(seedN ^ block)). */
int32_t mb_als_init_factors(int64_t seed, int32_t side, int32_t block, int32_t rank, int64_t count, double* out);
/* The device-resident links of one side (the arrays of mb_als_links, ids narrowed to int32, on the device), restricted
 * to the `count` positions of `work`.  The ctx stream must see them filled. */
typedef struct mb_als_side {
    int64_t count;
    const int32_t* ids;
    const int64_t* offsets;
    const int32_t* partners;
    const float* ratings;
    const int32_t* work;
} mb_als_side;
/* The assembly alone: for every position p in side->work, the packed lower triangle of A_p (row-major, element (i, j) at
 * i (i + 1) / 2 + j, regularisation and YtY included) to the DEVICE array A_out + p * rank (rank + 1) / 2 and b_p to
 * b_out + p * rank.  Y: the fixed side's factors.  YtY (rank x rank) is read when implicit; NULL computes it from Y. */
int32_t mb_als_normal_equations(mb_ctx* ctx, const mb_als_side* side, const mb_block* Y, double lambda, double alpha,
                                int32_t implicit, const mb_block* YtY, double* A_out, double* b_out);
/* One half-step: row p of X gets x_p for every position p in side->work; other rows are left as they are.  YtY as above.
 * Blocking (the pivot check reads back one int). */
int32_t mb_als_update(mb_ctx* ctx, const mb_als_side* side, const mb_block* Y, double lambda, double alpha, int32_t implicit,
                      const mb_block* YtY, mb_block* X);
/* The whole loop on one device (:77-82): `iterations` times, products from users then users from products, YtY computed on
 * the device each half-step when implicit (mb_block_gramian), no host synchronisation between half-steps.  U and P hold
 * the initial factors on entry and the result on return; iterations <= 0 leaves them as they are.  Blocking. */
int32_t mb_als_train(mb_ctx* ctx, const mb_als_side* users, const mb_als_side* products, int32_t iterations, double lambda,
                     double alpha, int32_t implicit, mb_block* U, mb_block* P);
/* updateBlock (:292-382) on HOST arrays, for the JVM: n positions with offsets[n + 1] / partners / ratings as from
 * mb_als_links and ids[n]; Y: n_fixed x rank row-major; YtY: rank x rank row-major or NULL (computed when implicit);
 * X: n x rank row-major.  Uploads, solves and frees inside the call. */
int32_t mb_als_update_host(mb_ctx* ctx, int32_t rank, int64_t n_fixed, const double* Y, int64_t n, const int64_t* ids,
                           const int64_t* offsets, const int32_t* partners, const float* ratings, double lambda,
                           double alpha, int32_t implicit, const double* YtY, double* X);
/* CoordinateMatrix.toDenseVecMatrix (matrix/CoordinateMatrix.scala:51-64): out (a row-major fp64 view) is zeroed and
 * gets out(row_pos[e], cols[e]) = values[e] from HOST arrays.  A repeated (row, col) is MB_ERR_INVALID_ARG
 * "requirement failed: Found duplicate indices: j." before anything is written, as Vectors.sparse fails. */
int32_t mb_coo_to_dense_rows(mb_ctx* ctx, int64_t nnz, const int32_t* row_pos, const int32_t* cols, const float* values,
                             mb_block* out);

/* ---- a11: MTUtils.randomDenVecMatrix / randomBlockMatrix input generation
 *      (utils/MTUtils.scala:34-73, rdd/RandomRDD.scala:28-101, utils/RandomDataGenerator.scala:53-65,113-131).
 * Fills `count` consecutive values of partition stream `partition_seed` (one XORShift stream per
 * RDD partition), bit-exact with UniformGenerator(lo,hi).nextValue(), starting at value index
 * `first` of that stream, written into blk in the order the reference fills it
 * (row_major=1: DenseVecMatrix rows, Array.fill(cols); row_major=0: BDM.create column-major). */
int32_t mb_fill_uniform(mb_ctx* ctx, mb_block* blk, int64_t partition_seed, int64_t first,
                        double lo, double hi, int32_t row_major);
/* StandardNormalGenerator(mean, variance) (utils/RandomDataGenerator.scala:70-82, rdd/RandomRDD.scala:70-112): fills blk
 * with the first rows * cols values of partition stream `partition_seed`, bit-exact with nextValue() =
 * mean + sqrt(variance) * nextGaussian(), in the order of mb_fill_uniform's `row_major` (rows one after another, so one
 * stream runs across rows and a pair of Gaussians may straddle two rows; or BDM.create column-major).  nextGaussian is
 * java.util.Random's polar method over XORShiftRandom.next (:113-131): attempt a takes nextDouble positions 2a and 2a + 1,
 * v = 2u - 1, s = v1*v1 + v2*v2, rejected when s >= 1 or s == 0, else m = StrictMath.sqrt(-2 * StrictMath.log(s) / s)
 * (fdlibm's log) and the attempt gives v1*m, then v2*m.  Each multiply and add is rounded separately; sqrt(variance) is
 * one correctly rounded value, so variance < 0 or NaN gives NaN everywhere and variance == 0 gives mean + (+-0.0).  The
 * generator starts fresh: no cached value comes in, and an odd count drops the last one.  fp64 blocks only (a view may
 * be strided; nothing outside it is written).  positions_out (may be NULL) receives 2A, the nextDouble positions the
 * values consumed, A being the index of the last attempt used plus one.  Blocking (see MB_NORMAL_TILE_ATTEMPTS).
 * More than 2^39 stream positions counted is MB_ERR_UNSUPPORTED. */
int32_t mb_fill_normal(mb_ctx* ctx, mb_block* blk, int64_t partition_seed, double mean, double variance, int32_t row_major,
                       int64_t* positions_out);
/* mb_fill_normal's three passes.  The attempts are cut into tiles of MB_NORMAL_TILE_ATTEMPTS; a count pass counts the
 * accepted attempts of a range of tiles, a scan turns the counts into prefixes, and a write pass regenerates the tiles that
 * hold needed pairs.  With pairs = ceil(n / 2), the first round counts
 *   ceil(ceil(pairs * 4.0 / 3.141592653589793) / MB_NORMAL_TILE_ATTEMPTS) tiles
 * (the product and the quotient in double arithmetic).  While the accepted attempts of the tiles counted fall short of
 * pairs by d > 0, a further round counts the next ceil(ceil(d * 4.0 / 3.141592653589793) / MB_NORMAL_TILE_ATTEMPTS)
 * tiles.  Each round is two kernel launches and one stream synchronisation, the write pass one launch (and one more
 * synchronisation for positions_out).  The budget never changes a result. */
#define MB_NORMAL_TILE_ATTEMPTS 32768
/* Host-side pieces of the same generator (pure integer logic, exported for the host mirror):
 * MTUtils.hashSeed (MurmurHash3.bytesHash over a 64-byte buffer) and the per-partition seeds
 * = successive java.util.Random(seed).nextLong() (rdd/RandomRDD.scala:28-45). */
int64_t mb_hash_seed(int64_t seed);
int32_t mb_partition_seeds(int64_t seed, int32_t num_partitions, int64_t* seeds_out);

/* ---- f6: sparse blocks (matrix/Matrices.scala:57-173, matrix/LibMatrixMult.scala, matrix/SubMatrix.scala:87-119).
 * A sparse block is CSC on the device: colptr int32[cols+1], rowidx int32[nnz], values f64[nnz], nnz < 2^31, row indices
 * strictly increasing within each column.  The reference's SparseMatrix (one SparseVector per column) accepts unsorted or
 * repeated indices unchecked; here they are MB_ERR_INVALID_ARG.  Products write a dense fp64 block or view; every output
 * element is summed by one thread in the reference loop's order with separate multiplies and adds, so results are bitwise
 * reproducible.  accumulate != 0: C := C + P, the complete product P added once (reduceByKey(add), BlockMatrix.scala:177). */
/* The structure checks of mb_sparse_upload on host arrays: colptr from 0 to nnz without decreasing, rows in [0, rows)
 * and strictly increasing within each column.  Pure logic; MB_ERR_INVALID_ARG with the first violation. */
int32_t mb_sparse_check(int32_t rows, int32_t cols, const int32_t* colptr, const int32_t* rowidx);
/* A handle over caller-owned device arrays (like mb_block_wrap: torch owns the memory, NCCL can move it).  The contents
 * are not read here; the caller guarantees the structure (e.g. a block that passed mb_sparse_check, or one that
 * mb_fill_sparse_uniform is about to write). */
int32_t mb_sparse_wrap(mb_ctx* ctx, int32_t rows, int32_t cols, int64_t nnz, void* colptr, void* rowidx, void* values,
                       mb_sparse** out);
/* Host CSC -> a library-owned device block, after mb_sparse_check.  nnz = colptr[cols].  Blocking. */
int32_t mb_sparse_upload(mb_ctx* ctx, int32_t rows, int32_t cols, const int32_t* colptr, const int32_t* rowidx,
                         const double* values, mb_sparse** out);
/* Device -> host arrays of cols+1, nnz and nnz elements.  Blocking. */
int32_t mb_sparse_download(mb_ctx* ctx, const mb_sparse* S, int32_t* colptr, int32_t* rowidx, double* values);
int32_t mb_sparse_info(const mb_sparse* S, int32_t* rows, int32_t* cols, int64_t* nnz);
/* A library-owned block with room for nnz entries (contents undefined until mb_fill_sparse_uniform or a copy writes them),
 * for callers that own no device memory of their own (the C++ mirror, the JVM). */
int32_t mb_sparse_alloc(mb_ctx* ctx, int32_t rows, int32_t cols, int64_t nnz, mb_sparse** out);
int32_t mb_sparse_free(mb_ctx* ctx, mb_sparse* S);
/* The scalar ops of a sparse SubMatrix (SubMatrix.scala:52-58, 71-85, 121-129): a new library-owned block with S's
 * structure whose stored values are v + b, v - b, v * b or v / b (op = MB_SPARSE_ADD / _SUB / _MUL / _DIV), computed by the
 * dense element-wise kernels; only the stored values change, as in the reference. */
#define MB_SPARSE_ADD 0
#define MB_SPARSE_SUB 1
#define MB_SPARSE_MUL 2
#define MB_SPARSE_DIV 3
int32_t mb_sparse_values_op(mb_ctx* ctx, const mb_sparse* S, int32_t op, double b, mb_sparse** out);
/* SparseMatrix.toDense (Matrices.scala:106-119) into a dense fp64 block or view of the same shape. */
int32_t mb_sparse_to_dense(mb_ctx* ctx, const mb_sparse* S, mb_block* out);
/* LibMatrixMult.multDenseSparse (LibMatrixMult.scala:15-41): C [+]= A * B for a dense view A.  C(:, j) sums B's column j
 * in stored order; a column holding exactly one value equal to 1.0 copies the A column (:28-29). */
int32_t mb_spmm_dense_sparse(mb_ctx* ctx, const mb_block* A, const mb_sparse* B, mb_block* C, int32_t accumulate);
/* LibMatrixMult.multSparseDense (:43-77): C [+]= A * B for a dense view B, C(r, i) summed over k ascending.  The reference
 * reads B(bi + k, i) where it means B(bk + k, i) (:60) and is right only for K <= 32 and N <= 32; this is the true product,
 * bit-identical to the corrected loop.  The first call builds a CSR copy of A on the device and keeps it with the handle
 * (about 12 * nnz + 4 * rows bytes, freed by mb_sparse_free). */
int32_t mb_spmm_sparse_dense(mb_ctx* ctx, mb_sparse* A, const mb_block* B, mb_block* C, int32_t accumulate);
/* SparseMatrix.multiply (Matrices.scala:129-152): C [+]= A * B, both sparse, the result dense. */
int32_t mb_spgemm_dense_out(mb_ctx* ctx, const mb_sparse* A, const mb_sparse* B, mb_block* C, int32_t accumulate);
/* The column count and the checks of a sparse randomBlockMatrix (SparseMatrix.rand, Matrices.scala:157-173):
 * s = (int)(cols * density) with the JVM's double product and truncation.  density <= 0 (or NaN) and s > rows (where the
 * reference's sampling loop never ends) are MB_ERR_INVALID_ARG.  Pure logic. */
int32_t mb_sparse_column_count(int32_t rows, int32_t cols, double density, int32_t* s_out);
/* The deterministic sparse generator of block `partition_seed` (the dense generator's per-block seed) into a block wrapped
 * over preallocated arrays with nnz = s * cols: values = positions [0, s*cols) of the block's XORShift stream (U[0,1),
 * column j taking [j*s, (j+1)*s)); column j's rows by selection sampling over positions [s*cols + j*rows, +rows):
 * exactly s sorted rows, every s-subset equally likely.  rows * cols draws per block whatever the density. */
int32_t mb_fill_sparse_uniform(mb_ctx* ctx, mb_sparse* S, int64_t partition_seed);

/* ---- SparseVecMatrix (matrix/SparseVecMatrix.scala).  A row shard (nloc rows of nCols columns) is CSR, held as the
 *      CSC handle of its transpose: an mb_sparse with rows = nCols and cols = nloc, whose colptr is the row pointer array
 *      and whose rowidx holds each row's column ids, strictly increasing (mb_sparse_check applies unchanged).
 *      toDenseVecMatrix (:56-65) is mb_sparse_to_dense into the transposed view of a row-major shard. ---- */
/* Row bins of mb_spvec_multiply by a row's product count u = sum over its stored k of nnz(B(k, :)): u <= WARP_BOUND is
 * one warp with a shared-memory hash, u <= CTA_BOUND one CTA with a larger hash, anything above one CTA walking windows
 * of MB_SPVEC_WINDOW columns.  The bin never changes a result. */
#define MB_SPVEC_WARP_BOUND 256
#define MB_SPVEC_CTA_BOUND  4096
#define MB_SPVEC_WINDOW     16384
/* multiplySparse (:22-50): C = A * B row by row.  A: the shard of A (handle rows = A.nCols), B: all of B laid out as one CSR
 * over row ids [0, B.nRows) (handle cols = B.nRows).  *out receives a new library-owned handle of C's rows in the same
 * form (rows = B.nCols, cols = A's local rows), columns ascending within each row; free it with mb_sparse_free.
 * Arithmetic: a = (float)A(i,k), b = (float)B(k,j), p = a * b in float32; C(i,j) is the first product of the row's k order
 * (A's stored order, k ascending), every later one added in float32, separately rounded, no flush to zero.  Entries are
 * the structural product: every (i, j) with at least one k stored on both sides, stored zeros and cancellations included.
 * The float32 results are stored widened to double in the values array (exact), so mb_sparse_download, mb_sparse_to_dense
 * and mb_sparse_free apply unchanged.  A.nCols != B.nRows is MB_ERR_DIM_MISMATCH (the reference drops the unmatched k);
 * more than 2^31 - 1 output entries is MB_ERR_UNSUPPORTED naming the count.  Synchronises the stream twice (bin sizes,
 * total count). */
int32_t mb_spvec_multiply(mb_ctx* ctx, const mb_sparse* A, const mb_sparse* B, mb_sparse** out);
/* The same product on HOST CSR arrays, for callers holding rows on the host (the JVM, the C++ mirror): A is a_rows rows of
 * k columns (a_rowptr[a_rows + 1], a_colidx, a_values), B is k rows of n columns (absent row ids empty).  Both are checked
 * as mb_sparse_upload checks a block (MB_ERR_INVALID_ARG on unsorted or repeated columns).  Uploads, multiplies and frees
 * the inputs; *out receives a library-owned handle of C's rows as from mb_spvec_multiply.  Blocking. */
int32_t mb_spvec_multiply_host(mb_ctx* ctx, int32_t a_rows, int32_t k, const int32_t* a_rowptr, const int32_t* a_colidx,
                               const double* a_values, int32_t n, const int32_t* b_rowptr, const int32_t* b_colidx,
                               const double* b_values, mb_sparse** out);
/* The entries of a row handle (from mb_spvec_multiply / _host) as HOST COO arrays of nnz elements (mb_sparse_info): the
 * local row position, the column and the float32 value, rows ascending and columns ascending within a row.  Blocking. */
int32_t mb_spvec_coo(mb_ctx* ctx, const mb_sparse* C, int32_t* rows_out, int32_t* cols_out, float* values_out);
/* DenseVecMatrix.toSparseVecMatrix (DenseVecMatrix.scala:1333-1353): the rows of an fp64 view (one matrix row per shard
 * row, any ld) to a new library-owned handle (rows = view cols, cols = view rows) keeping the entries v != 0.0 in column
 * order: NaN is kept, +-0.0 dropped.  Blocking (one synchronisation to size the result). */
int32_t mb_dense_rows_to_sparse(mb_ctx* ctx, const mb_block* rows, mb_sparse** out);
/* randomSpaVecMatrix (utils/MTUtils.scala:75-85, rdd/RandomRDD.scala:136-159) for one partition of P rows: S (rows =
 * nColumns, cols = P, nnz = s * P with s from mb_sparse_column_count(nColumns, nColumns, density)) gets
 *   values: positions [0, s*P) of the partition's XORShift stream as U[lo, hi) (row r takes [r*s, (r+1)*s)), bit-identical
 *           to randomDenVecMatrix's stream for the same partition seed;
 *   columns: ONE sorted set of s distinct columns shared by all P rows, as in the reference, drawn by selection sampling
 *           (mb_fill_sparse_uniform's sampler) over positions [s*P, s*P + nColumns) of the same stream.
 * The reference draws the set from an unseeded java.util.Random; here it is a function of (seed, partition). */
int32_t mb_fill_spvec_uniform(mb_ctx* ctx, mb_sparse* S, int64_t partition_seed, double lo, double hi);
/* randomSpaVecMatrix with StandardNormalGenerator(mean, variance): S as for mb_fill_spvec_uniform, its values the first
 * s * P values of mb_fill_normal's stream for the partition (row r takes [r*s, (r+1)*s)).  For both entries the one column
 * set is drawn from the stream positions right after those the values consumed: [2A, 2A + nColumns) here, 2A as
 * mb_fill_normal's positions_out; [s*P, s*P + nColumns) for the uniform values, which consume exactly s*P positions.
 * Blocking. */
int32_t mb_fill_spvec_normal(mb_ctx* ctx, mb_sparse* S, int64_t partition_seed, double mean, double variance);

/* ---- PageRank (examples/PageRank.scala).  The link matrix is held as the in-link CSR of the target pages: the CSC handle
 *      of its transpose, an mb_sparse with rows = n (source pages) and cols = the number of target rows, whose colptr is the
 *      row pointer array and whose rowidx holds each target's sources, strictly increasing (mb_sparse_check applies).
 *      One iteration of the example (links.multiply(ranks) over the 1 x numBlocks block grid of
 *      linkRows.transpose(numBlocks).multiply(0.85), BlockMatrix.scala:240-259, then .reduce(add).add(0.15 * ones)) is,
 *      for every target row i,
 *        y_i = fl(fl(P_0 + P_1 + ...) + addend),
 *      P_s = 0.0 + fl(w_ij x_j) + ... over the stored sources j in [s * seg_len, (s + 1) * seg_len), ascending, each
 *      multiply and add rounded separately (F2J dgemv per block column), the partials folded left in segment order.  With
 *      finite x >= 0 the terms of the non-links the dense blocks hold are +0.0, so the result is the dense composition's
 *      bit for bit.  Errors: seg_len <= 0 is MB_ERR_INVALID_ARG; x or y of the wrong length MB_ERR_DIM_MISMATCH. ---- */
/* In-degree above which a target row gets a warp of its own instead of one lane.  The bin never changes a result. */
#define MB_PAGERANK_LIGHT_BOUND 256
/* Pure host logic (loadLinksMatrix :13-27 and transpose, DenseVecMatrix.scala:1420-1436): the in-link CSR of targets
 * [t0, t1) from the link rows in source-major CSR.  Row r is source page ids[r] (in [0, n), distinct) with targets
 * targets[rowptr[r] .. rowptr[r + 1]) (strictly increasing, in [0, n)) and values values[...].  Writes
 *   in_rowptr_out[t1 - t0 + 1]        target t0 + k holds entries [in_rowptr_out[k], in_rowptr_out[k + 1])
 *   sources_out[nnz], weights_out[nnz] the source ids ascending (a stable counting sort by target over the rows taken
 *                                      in ascending source order) and fl(value * damping)
 * with nnz (<= rowptr[num_rows]) in *nnz_out.  Anything out of range is MB_ERR_INVALID_ARG naming it; more than
 * 2^31 - 1 entries is MB_ERR_UNSUPPORTED. */
int32_t mb_pagerank_links(int32_t n, int64_t num_rows, const int64_t* ids, const int64_t* rowptr, const int32_t* targets,
                          const double* values, int32_t t0, int32_t t1, double damping, int32_t* in_rowptr_out,
                          int32_t* sources_out, double* weights_out, int64_t* nnz_out);
/* One iteration: y (in_links->cols x 1) = the step above applied to x (in_links->rows x 1).  x and y are contiguous fp64
 * blocks of one column; y must not overlap x.  The first step or train call on a handle bins its rows by in-degree and
 * keeps the list with the handle (one stream synchronisation); later calls only enqueue. */
int32_t mb_pagerank_step(mb_ctx* ctx, mb_sparse* in_links, const mb_block* x, int64_t seg_len, double addend, mb_block* y);
/* The whole loop on one device: `iterations` steps of a square in_links (rows == cols == n), ping-ponging x_inout (n x 1)
 * and one scratch vector with no host synchronisation between steps; x_inout holds the initial ranks on entry and the
 * result on return.  iterations <= 0 leaves x_inout as it is.  Blocking. */
int32_t mb_pagerank_train(mb_ctx* ctx, mb_sparse* in_links, int64_t seg_len, double addend, int32_t iterations,
                          mb_block* x_inout);
/* The same loop on HOST arrays, for callers holding the link rows on the host (the JVM, the C++ mirror): the link rows as
 * for mb_pagerank_links over all n targets and the damping factor; ranks_inout (n doubles) holds the initial ranks on
 * entry and the result on return.  Builds the in-links, uploads, runs and frees inside the call.  Blocking. */
int32_t mb_pagerank_host(mb_ctx* ctx, int32_t n, int64_t num_rows, const int64_t* ids, const int64_t* rowptr,
                         const int32_t* targets, const double* values, double damping, int64_t seg_len, double addend,
                         int32_t iterations, double* ranks_inout);

/* ---- The NeuralNetwork example (examples/NeuralNetwork.scala): mini-batch SGD on a two-layer sigmoid network with ten
 *      output units.  For the selected row blocks X_b (r_b x V) of one iteration, with W1 (V x H) and W2 (H x 10):
 *        Z1_b = X_b W1 (:222-225); A1_b = sigmoid(Z1_b), A2_b = sigmoid(A1_b W2) (:226-231);
 *        D2_b = (1 - A2_b) A2_b (A2_b - onehot(labels_b)) (:119-128, :152-162); D1_b = (1 - A1_b) A1_b (D2_b W2^T) (:240-241);
 *        dW2 = sum_b fl(scale * A1_b^T D2_b), dW1 = sum_b fl(scale * X_b^T D1_b), blocks in the order given
 *        (computeWeightUpd :171-183 with scale = learningRate / batchSize; the reference's treeReduce order is not fixed).
 *      Z1_b and X_b^T D1_b run on the fp64 DMMA GEMM; everything between them is one fused kernel per block, so the
 *      activations never reach device memory and the hidden layer is written once (Z1) and replaced once (D1).  XT[b] is
 *      X_b^T materialised (V x r_b, column-major): with it, X_b^T D1_b is split over its r_b-long inner dimension into
 *      chunks that run as entries of one grouped launch, which fills the SMs where one GEMM of (V/128) x (H/128) tiles
 *      cannot.  XT, or any XT[b], may be NULL, and an XT[b] that is not 16-byte aligned with an even leading dimension (an
 *      odd V) is not used: that block's product is then one transposed-A GEMM over X_b.  W1, W2 and the outputs are
 *      column-major fp64 blocks; a bf16 or fp32 block anywhere is MB_ERR_UNSUPPORTED, a shape that does not fit
 *      MB_ERR_DIM_MISMATCH.  Sums run in a fixed order: the same call gives the same bits.  Nothing here synchronises with
 *      the host; device temporaries are returned in stream order. ---- */
/* `count` labels of one block (DistributedIntVector piece, :71-80) as a device array for the two entries below.  A label
 * outside 0..9 is MB_ERR_INVALID_ARG naming its row (ArrayIndexOutOfBounds in computeOutputError on the JVM). */
int32_t mb_nn_labels_upload(mb_ctx* ctx, const int32_t* labels, int64_t count, void** labels_out);
int32_t mb_nn_labels_free(mb_ctx* ctx, void* labels);
/* The two scaled gradient sums of the nsel blocks one rank holds: dW1_out (V x H) and dW2_out (H x 10).  labels[b] comes
 * from mb_nn_labels_upload and holds X[b]->rows labels.  D1_out is NULL or nsel blocks (each NULL or r_b x H, column-major)
 * that receive D1_b; without one, D1_b replaces Z1_b in the call's workspace. */
int32_t mb_nn_gradient(mb_ctx* ctx, const mb_block* const* X, const mb_block* const* XT, const void* const* labels,
                       int32_t nsel, const mb_block* W1, const mb_block* W2, double scale, mb_block* dW1_out,
                       mb_block* dW2_out, mb_block* const* D1_out);
/* One iteration on one rank (:219-248): the same, then W1 -= dW1 and W2 -= dW2, both from the W2 before the step.  The
 * weights stay on the device between steps. */
int32_t mb_nn_step(mb_ctx* ctx, const mb_block* const* X, const mb_block* const* XT, const void* const* labels, int32_t nsel,
                   mb_block* W1, mb_block* W2, double scale);

/* ---- a7/a8: strategy + partitioning (pure integer logic) --------------------------------- */
/* MTUtils.splitMethod(m,k,n,cores) (utils/MTUtils.scala:150-175, dimToSplit :204-213) */
int32_t mb_choose_split(int64_t m, int64_t k, int64_t n, int32_t cores, int32_t out_mkn[3]);
/* DenseVecMatrix.multiply(other,cores,broadcastThreshold) chooser (matrix/DenseVecMatrix.scala:196-231,
 * matrix/BlockMatrix.scala:87-122).  other_is_block selects the `case that: BlockMatrix` arm.
 * Returns strategy in *strategy: 0 = broadcast B (this.multiply(that.toBreeze())),
 * 1 = broadcast A (the reference's quirk arm), 2 = shuffle with out_mkn. */
int32_t mb_choose_strategy(int64_t a_rows, int64_t a_cols, int64_t b_cols, int32_t cores,
                           int32_t broadcast_threshold_mb, int32_t other_is_block,
                           int32_t* strategy, int32_t out_mkn[3]);
/* MatrixMultPartitioner (rdd/MatrixMultPartitioner.scala:12-22) with the seq formula of
 * matrix/BlockMatrix.scala:163,168: seq = i*n*k + j*k + kk. */
int32_t mb_mult_partition(int32_t i, int32_t j, int32_t kk, int32_t m, int32_t k, int32_t n);
/* MatrixElemOpPartitioner (rdd/MatrixElemOpPartitioner.scala:16) */
int32_t mb_elem_partition(int32_t row, int32_t col, int32_t blks_by_col);
/* ceil-based block sizing (matrix/BlockMatrix.scala:73-74, matrix/DenseVecMatrix.scala:1091-1094):
 * block length = ceil(total/parts); actual number of blocks = ceil(total/block_len). */
int32_t mb_block_len(int64_t total, int32_t parts, int32_t* block_len, int32_t* actual_parts);

/* ---- a3/a4: BlockMatrix.multiply(other: BlockMatrix) on ONE device
 *      (matrix/BlockMatrix.scala:149-186): all m*k*n block products in seq order, the k partials of
 *      each C tile accumulated in place.  A_tiles[i*k+kk], B_tiles[kk*n+j], C_tiles[i*n+j]
 *      (MatrixElemOpPartitioner order).  Multi-GPU sharding of the seq list is done by the host
 *      (marlin_b200.matrix.BlockMatrix) with one process per GPU. */
int32_t mb_matmul_blocked(mb_ctx* ctx, mb_block* const* A_tiles, mb_block* const* B_tiles,
                          int32_t m, int32_t k, int32_t n, mb_block* const* C_tiles);
/* The share of that multiply one rank runs: only the C blocks listed in c_ids (c = i*n + j), each with its full
 * kk-sum.  Tile slots this rank does not need may be NULL.  fp64 'N' blocks run as ONE persistent grouped launch
 * (K loop concatenated over kk, no C read-modify-write); anything else falls back to per-product launches. */
int32_t mb_matmul_blocked_subset(mb_ctx* ctx, mb_block* const* A_tiles, mb_block* const* B_tiles,
                                 int32_t m, int32_t k, int32_t n, mb_block* const* C_tiles,
                                 const int32_t* c_ids, int32_t num_c);

/* The same multiply for JVM-held blocks (HOST column-major fp64 arrays in, host arrays out): the entry a
 * `BlockMatrix.multiply` whose SubMatrix data still lives on the heap would bind.  A_host[i*k+kk] is the packed
 * (row_len[i] x k_len[kk]) tile, B_host[kk*n+j] the (k_len[kk] x col_len[j]) tile, C_host[i*n+j] receives the
 * (row_len[i] x col_len[j]) result.  Uploads, the m*k*n DMMA products (seq order, kk accumulated in the epilogue)
 * and downloads are pipelined on separate streams: tiles are uploaded in first-use order and every C tile
 * starts its D2H as soon as its last partial is done.  Pinned host memory gives full PCIe overlap; pageable
 * memory still works (the copies just serialise).  This is the end-to-end path bench.py times at N=1. */
int32_t mb_matmul_blocked_host(mb_ctx* ctx, const double* const* A_host, const double* const* B_host,
                               int32_t m, int32_t k, int32_t n, const int32_t* row_len, const int32_t* k_len,
                               const int32_t* col_len, double* const* C_host);

/* a5: DenseVecMatrix.multiply(B: BDM[Double]) (matrix/DenseVecMatrix.scala:1660-1680) for the row shard one process
 * holds: C_rows = A_rows * B.  A_rows / C_rows are row-major shards (transposed views of the column-major array
 * underneath), B is the broadcast matrix; the rows never change GPU, so N ranks run N independent calls. */
int32_t mb_matmul_rowsharded(mb_ctx* ctx, const mb_block* A_rows, const mb_block* B, mb_block* C_rows);
/* The same for JVM-held rows: A_host = the shard's rows back to back (row-major, k doubles per row: the packed
 * `rowsMat` of :1672-1675), B_host = column-major k x n, C_host receives rows x n row-major.  Row chunks of ~256 MiB
 * are pipelined over three streams (H2D of chunk c+1, the DMMA product of chunk c, D2H of chunk c-1). */
int32_t mb_matmul_rowsharded_host(mb_ctx* ctx, const double* A_host, int64_t rows, int32_t k, const double* B_host,
                                  int32_t n, double* C_host);

/* ---- peer memory: NVLink P2P between the per-GPU processes of one box (CUDA IPC) ------------------------------
 * Replaces the shuffle transport of the multiply (matrix/BlockMatrix.scala:161-177): a rank maps the tile buffers
 * of the others once, pulls the tiles it needs with copy-engine DMA (mb_memcpy_async on a side stream) and lets its
 * GEMM epilogue store partial products directly into the reducing rank's memory (pass a peer pointer as C).
 * Ordering between processes uses stream-ordered flags (monotonic epochs) living in exported device memory. */
int32_t mb_ipc_export(mb_ctx* ctx, const void* device_ptr, uint8_t handle_out[64], int64_t* offset_out,
                      int64_t* alloc_bytes_out);
int32_t mb_ipc_open(mb_ctx* ctx, const uint8_t handle[64], void** base_out);     /* cached per handle */
int32_t mb_ipc_close_all(mb_ctx* ctx);
int32_t mb_flags_alloc(mb_ctx* ctx, int32_t count, void** flags_out);            /* zeroed uint64[count], cudaMalloc'd */
int32_t mb_flags_free(mb_ctx* ctx, void* flags);
int32_t mb_flag_signal(mb_ctx* ctx, void* flag, int64_t value);   /* on the ctx stream: release-store (system scope) */
int32_t mb_flag_wait(mb_ctx* ctx, const void* flag, int64_t value); /* on the ctx stream: wait until *flag >= value */
int32_t mb_memcpy_async(mb_ctx* ctx, void* dst, const void* src, int64_t bytes);   /* D2D (local or peer) on the ctx stream */

/* ---- (e) BlockMatrix.multiply across the GPUs of one box, entirely behind this ABI ---------------------------------
 * One process (or thread with its own ctx) per GPU.  mb_comm is the analogue of the executors of one SparkContext:
 * created once, collectively, by `world` ranks that pass the same `session` string (unique per communicator: it names a
 * POSIX shared-memory segment used for rendezvous and per-call tile directories — no network, no torch, no MPI).
 * mb_matmul_blocked_dist is the whole of matrix/BlockMatrix.scala:159-178 — MatrixMultPartitioner mapping
 * (seq = i*n*k + j*k + kk dealt to ranks in contiguous ranges: mb_dist_plan), tile replication (NVLink peer-memory
 * pulls overlapped with the products), the m*k*n DMMA block products (one persistent launch per rank; two where a k
 * partial crosses GPUs) and the reduceByKey of the k partials (reduce-scatter by the GEMM epilogues between two holders,
 * staged adds otherwise).
 * Every rank calls it with the same m, k, n, lengths and owner maps; A_tiles[i*k+kk] / B_tiles[kk*n+j] are non-NULL
 * exactly where the owner map names this rank; C_tiles[i*n+j] must be a preallocated (row_len[i] x col_len[j]) block
 * (F64, or F32 for BF16 inputs) wherever mb_dist_plan's c_owner names this rank, and receives the finished tile there.
 * Asynchronous like every other compute entry: ordered on the ctx stream.  Flags between the processes are stream memory
 * operations and peer stores, never kernels (nothing the resident GEMM waits for needs an SM); in-kernel waits are bounded
 * by MARLIN_B200_TIMEOUT_S, host-side waits too (then the communicator aborts itself and the call returns MB_ERR_TIMEOUT).
 * Give every stream its own hardware queue: CUDA_DEVICE_MAX_CONNECTIONS=32 before the CUDA context is created. */
typedef struct mb_comm mb_comm;
#define MB_ERR_TIMEOUT       -7   /* a peer did not answer within MARLIN_B200_TIMEOUT_S (default 120 s) -> RuntimeException */
int32_t mb_comm_init(mb_ctx* ctx, int32_t rank, int32_t world, const char* session, mb_comm** out);
int32_t mb_comm_destroy(mb_comm* comm);
int32_t mb_comm_rank(const mb_comm* comm);
int32_t mb_comm_world(const mb_comm* comm);
int32_t mb_comm_barrier(mb_comm* comm);            /* host-side barrier of the ranks */
int32_t mb_comm_abort(mb_comm* comm);              /* release every wait queued on this rank (results garbage); the comm is dead */
int32_t mb_comm_check(mb_comm* comm);              /* MB_ERR_TIMEOUT if a device-side wait for a peer ever gave up */
/* MatrixMultPartitioner + placement: product seq -> rank (m*k*n entries) and C tile -> owning rank (m*n entries). */
int32_t mb_dist_plan(int32_t m, int32_t k, int32_t n, int32_t world, int32_t* product_rank_out, int32_t* c_owner_out);
int32_t mb_matmul_blocked_dist(mb_comm* comm, mb_block* const* A_tiles, const int32_t* a_owner,
                               mb_block* const* B_tiles, const int32_t* b_owner, int32_t m, int32_t k, int32_t n,
                               const int32_t* row_len, const int32_t* k_len, const int32_t* col_len, int32_t dtype,
                               mb_block* const* C_tiles);

/* The same multiply END TO END with HOST tiles (what bench.py reports as e2e at N > 1): every input tile is uploaded by
 * ONE of the ranks that need it (a_home / b_home; mb_dist_host_homes spreads them over the PCIe links) and pulled over
 * NVLink by the others, band by band; one grouped DMMA launch per rank starts on the first bands; the two holders of a
 * k-split C tile each reduce and download a checkerboard of its sub-blocks, hidden behind the rest of the GEMM.
 * A_host / B_host: packed column-major tiles, non-NULL where homed; C_host[i*n+j]: the packed host tile, non-NULL on
 * every rank that computes a partial of it (use one mb_host_alloc_shared array per tile so that the ranks fill one copy).
 * fp64, at most two holders per C tile.  Blocking. */
int32_t mb_dist_host_homes(int32_t m, int32_t k, int32_t n, int32_t world, int32_t* a_home, int32_t* b_home);
int32_t mb_matmul_blocked_dist_host(mb_comm* comm, const double* const* A_host, const int32_t* a_home,
                                    const double* const* B_host, const int32_t* b_home, int32_t m, int32_t k, int32_t n,
                                    const int32_t* row_len, const int32_t* k_len, const int32_t* col_len,
                                    double* const* C_host);
/* Pinned host memory shared by the processes of one box (POSIX shm `name` + cudaHostRegister). */
int32_t mb_host_alloc_shared(const char* name, int64_t bytes, void** out);
int32_t mb_host_free_shared(const char* name, void* ptr, int64_t bytes, int32_t unlink_name);

/* ---- f3: matrix text files, written on the device (matrix/DenseVecMatrix.scala:1042-1046, matrix/BlockMatrix.scala:550-555).
 * Every value is printed as java.lang.Double.toString prints it: the shortest decimal that reads back as the same double
 * (the closest one when several are as short), plain for 1e-3 <= |v| < 1e7, d.dddE[-]n otherwise, NaN, Infinity,
 * -Infinity, -0.0.  Where the JVM picks a closer two-digit form of a one-digit decimal, this keeps the shortest one:
 * Double.MIN_VALUE is 5.0E-324 (4.9E-324 on the JVM).  fp32 and bf16 blocks are widened to double first.  The text is
 * formatted in chunks of at most MB_TEXT_CHUNK_VALUES values, two kernel launches each, and streamed to the file through
 * pinned host memory; a view that holds no values is formatted on the host.  Each entry writes one part file, truncating
 * it; a file that cannot be opened or written is MB_ERR_IO naming it.  Blocking. */
#define MB_TEXT_CHUNK_VALUES 2097152
/* DenseVecMatrix.saveToFileSystem's part file: `row_ids[r]:DenseVector(v, v, ...)` and a newline for each row r of the
 * shard `rows` (a rows x cols view, read row by row; a row with no columns is `id:DenseVector()`).  rows may be NULL: an
 * empty shard, an empty file.  row_ids: host int64[rows->rows]. */
int32_t mb_save_rows(mb_ctx* ctx, const mb_block* rows, const int64_t* row_ids, const char* path);
/* BlockMatrix.saveToFileSystem(path, "blockmatrix")'s part file: for block i, `r-c-rows-cols:v,v,...` and a newline, with
 * (r, c) = (block_rc[2i], block_rc[2i + 1]) and the values column by column. */
int32_t mb_save_blocks(mb_ctx* ctx, const mb_block* const* blocks, const int32_t* block_rc, int32_t count, const char* path);

/* ---- rows <-> blocks on device (matrix/DenseVecMatrix.scala:1084-1223, 1259-1328;
 *      matrix/BlockMatrix.scala:575-594): a DenseVecMatrix shard is a row-major (rows x cols)
 *      buffer, i.e. a transposed block; these are strided copies (mb_block_copy on views). */

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif /* MARLIN_B200_H */

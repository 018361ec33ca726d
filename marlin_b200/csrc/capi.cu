// C ABI of libmarlin_b200.so (see include/marlin_b200.h).  Context, block handles and dispatch.
// There is no CPU fallback anywhere in this file: without a CUDA device mb_init fails with
// MB_ERR_CUDA and no compute entry can be reached.
#include "../../include/marlin_b200.h"
#include "elementwise.h"
#include "gemm_f64.h"
#include "gemm_bf16.h"
#include "gemm_ozaki.h"
#include "blas12.h"
#include "factor.h"
#include "eigen.h"
#include "sparse.h"
#include "logistic.h"
#include "als.h"
#include "spvec.h"
#include "pagerank.h"
#include "mlp.h"
#include "norm.h"
#include "eigs.h"
#include "normal.h"
#include "text.h"

#include <cuda_runtime.h>
#include <cerrno>
#include <climits>
#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdlib>
#include <cstdio>
#include <cstring>
#include <new>
#include <atomic>
#include <memory>
#include <mutex>
#include <vector>

#include "internal.h"

namespace {

thread_local char g_err[512] = "";

int32_t new_block(mb_block** out) {
    *out = new (std::nothrow) mb_block();
    if (!*out) return fail(MB_ERR_OOM, "host allocation failed");
    return MB_OK;
}

// A new handle until its entry returns it: freed on every failure path, handed to *out by release() on success.
struct BlockFree { mb_ctx* ctx; void operator()(mb_block* b) const { mb_block_free(ctx, b); } };
struct SparseFree { mb_ctx* ctx; void operator()(mb_sparse* s) const { mb_sparse_free(ctx, s); } };
using BlockPtr = std::unique_ptr<mb_block, BlockFree>;
using SparsePtr = std::unique_ptr<mb_sparse, SparseFree>;

int32_t same_shape(const mb_block* a, const mb_block* b, const char* what) {
    if (a->rows != b->rows || a->cols != b->cols)
        return fail(MB_ERR_DIM_MISMATCH, "matrix dimension mismatch in %s: %dx%d vs %dx%d", what, a->rows, a->cols,
                    b->rows, b->cols);
    return MB_OK;
}

// The transpose of a block: a non-owning view of the same storage.
mb_block transposed(const mb_block& b) {
    mb_block t = b;
    t.owns = 0;
    std::swap(t.rows, t.cols);
    t.is_transpose = !b.is_transpose;
    return t;
}

// Element-wise kernels iterate in the output's storage order so the store side is contiguous: with a transposed output
// every operand is walked through its transpose.
mb_block in_out_order(const mb_block* b, const mb_block* out) { return out->is_transpose ? transposed(*b) : *b; }

int32_t binary_op(mb_ctx* ctx, int op, const mb_block* A, const mb_block* B, mb_block* out, const char* name) {
    MB_CTX(ctx);
    if (!A || !B || !out) return fail(MB_ERR_INVALID_ARG, "%s: null block", name);
    int32_t r = same_shape(A, B, name);
    if (r) return r;
    r = same_shape(A, out, name);
    if (r) return r;
    const bool all_f32 = A->dtype == MB_F32 && B->dtype == MB_F32 && out->dtype == MB_F32;
    if (!all_f32 && (A->dtype != MB_F64 || B->dtype != MB_F64 || out->dtype != MB_F64))
        return fail(MB_ERR_UNSUPPORTED, "%s: fp64 (or all-fp32) blocks only (convert bf16 blocks with mb_block_copy)", name);
    const mb_block a = in_out_order(A, out), b = in_out_order(B, out), o = in_out_order(out, out);
    if (all_f32) {
        MB_CUDA(mb::ew_binary_f32(op, a.rows, a.cols, reinterpret_cast<const float*>(elem_ptr(&a)), rs(&a), cs(&a),
                                  reinterpret_cast<const float*>(elem_ptr(&b)), rs(&b), cs(&b), reinterpret_cast<float*>(elem_ptr(&o)),
                                  rs(&o), cs(&o), ctx->stream));
        return MB_OK;
    }
    MB_CUDA(mb::ew_binary(op, a.rows, a.cols, f64_ptr(&a), rs(&a), cs(&a), f64_ptr(&b), rs(&b), cs(&b), f64_ptr(&o), rs(&o), cs(&o),
                          ctx->stream));
    return MB_OK;
}

int32_t unary_op(mb_ctx* ctx, int op, const mb_block* A, mb_block* out, double alpha, double beta, const char* name) {
    MB_CTX(ctx);
    if (!A || !out) return fail(MB_ERR_INVALID_ARG, "%s: null block", name);
    int32_t r = same_shape(A, out, name);
    if (r) return r;
    if (A->dtype != MB_F64 || out->dtype != MB_F64)
        return fail(MB_ERR_UNSUPPORTED, "%s: fp64 blocks only", name);
    const mb_block a = in_out_order(A, out), o = in_out_order(out, out);
    MB_CUDA(mb::ew_unary(op, a.rows, a.cols, f64_ptr(&a), rs(&a), cs(&a), f64_ptr(&o), rs(&o), cs(&o), alpha, beta, ctx->stream));
    return MB_OK;
}

// out (col-major packed or strided, same logical shape as `A` view) = A, with dtype conversion.
int32_t copy_convert(mb_ctx* ctx, const mb_block* A, mb_block* out) {
    const mb_block a = in_out_order(A, out), o = in_out_order(out, out);
    const int rows = a.rows, cols = a.cols;
    const long long ars = rs(&a), acs = cs(&a), ors = rs(&o), ocs = cs(&o);
    if (A->dtype == MB_F64 && out->dtype == MB_F64) {
        if (ars == 1 && ors == 1) {
            MB_CUDA(mb::ew_unary(mb::EW_COPY, rows, cols, f64_ptr(A), ars, acs, f64_ptr(out), ors, ocs, 1.0, 0.0, ctx->stream));
        } else if (acs == 1 && ors == 1) {
            // source is the transpose of a column-major (cols x rows, ld = ars) array
            MB_CUDA(mb::transpose_f64(f64_ptr(A), ars, f64_ptr(out), ocs, cols, rows, ctx->stream));
        } else {
            MB_CUDA(mb::ew_unary(mb::EW_COPY, rows, cols, f64_ptr(A), ars, acs, f64_ptr(out), ors, ocs, 1.0, 0.0, ctx->stream));
        }
    } else if (A->dtype == out->dtype && acs == 1 && ors == 1 && A->dtype == MB_BF16) {
        MB_CUDA(mb::transpose_b16(elem_ptr(A), ars, elem_ptr(out), ocs, cols, rows, ctx->stream));
    } else if (A->dtype == out->dtype && acs == 1 && ors == 1 && A->dtype == MB_F32) {
        MB_CUDA(mb::transpose_b32(elem_ptr(A), ars, elem_ptr(out), ocs, cols, rows, ctx->stream));
    } else {
        MB_CUDA(mb::convert_strided(A->dtype, out->dtype, rows, cols, elem_ptr(A), ars, acs, elem_ptr(out), ors, ocs, ctx->stream));
    }
    return MB_OK;
}


// A block with one column (or one row) read as a vector: element i lives at p[i * inc].
struct vec_view {
    double* p;
    long long inc;
    int len;
};
bool as_vector(const mb_block* b, vec_view* v) {
    if (b->dtype != MB_F64) return false;
    if (b->cols == 1) { v->len = b->rows; v->inc = rs(b); }
    else if (b->rows == 1) { v->len = b->cols; v->inc = cs(b); }
    else return false;
    v->p = f64_ptr(b);
    return true;
}

}  // namespace

int32_t mb_fail(int32_t code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

extern "C" {

const char* mb_last_error(void) { return g_err; }
const char* mb_version(void) { return "marlin_b200 0.1 (sm_90a)"; }

int32_t mb_init(int32_t device, mb_ctx** out) {
    if (!out) return fail(MB_ERR_INVALID_ARG, "mb_init: null out");
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0)
        return fail(MB_ERR_CUDA, "mb_init: no CUDA device (%s); marlin_b200 has no CPU fallback",
                    e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
    if (device < 0 || device >= count) return fail(MB_ERR_INVALID_ARG, "mb_init: device %d out of range [0,%d)", device, count);
    MB_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    MB_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
        return fail(MB_ERR_UNSUPPORTED, "mb_init: device %d is sm_%d%d; this library is built for sm_90a only", device,
                    prop.major, prop.minor);
    mb_ctx* ctx = new (std::nothrow) mb_ctx();
    if (!ctx) return fail(MB_ERR_OOM, "host allocation failed");
    ctx->device = device;
    ctx->num_sms = prop.multiProcessorCount;
    MB_CUDA(cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking));
    ctx->stream = ctx->own_stream;
    MB_CUDA(cudaMalloc(&ctx->scratch, sizeof(double) * std::max(mb::sum_scratch_doubles(), mb::dot_scratch_doubles())));
    MB_CUDA(cudaMallocHost(&ctx->host_scalar, sizeof(double)));
    MB_CUDA(cudaEventCreate(&ctx->ev0));
    MB_CUDA(cudaEventCreate(&ctx->ev1));
    *out = ctx;
    return MB_OK;
}

int32_t mb_shutdown(mb_ctx* ctx) {
    if (!ctx) return MB_OK;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    if (ctx->scratch) cudaFree(ctx->scratch);
    if (ctx->vec_ws) cudaFree(ctx->vec_ws);
    if (ctx->int_ws) cudaFree(ctx->int_ws);
    if (ctx->int_host) cudaFreeHost(ctx->int_host);
    if (ctx->host_scalar) cudaFreeHost(ctx->host_scalar);
    if (ctx->ev0) cudaEventDestroy(ctx->ev0);
    if (ctx->ev1) cudaEventDestroy(ctx->ev1);
    for (cudaEvent_t ev : ctx->events) cudaEventDestroy(ev);
    if (ctx->own_stream) cudaStreamDestroy(ctx->own_stream);
    if (ctx->h2d_stream) cudaStreamDestroy(ctx->h2d_stream);
    if (ctx->d2h_stream) cudaStreamDestroy(ctx->d2h_stream);
    if (ctx->workspace) cudaFree(ctx->workspace);
    if (ctx->ozaki_ws) cudaFree(ctx->ozaki_ws);
    delete ctx;
    return MB_OK;
}

int32_t mb_set_stream(mb_ctx* ctx, void* cuda_stream) {
    if (!ctx) return fail(MB_ERR_INVALID_ARG, "null context");
    ctx->stream = static_cast<cudaStream_t>(cuda_stream);
    return MB_OK;
}

int32_t mb_reset_stream(mb_ctx* ctx) {
    if (!ctx) return fail(MB_ERR_INVALID_ARG, "null context");
    ctx->stream = ctx->own_stream;
    return MB_OK;
}

int32_t mb_synchronize(mb_ctx* ctx) {
    MB_CTX(ctx);
    MB_CUDA(cudaStreamSynchronize(ctx->stream));
    return MB_OK;
}

int64_t mb_launch_count(mb_ctx* ctx) { return ctx ? (int64_t)ctx->launches.load() : 0; }

int32_t mb_timer_start(mb_ctx* ctx) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    MB_CUDA(cudaEventRecord(ctx->ev0, ctx->stream));
    return MB_OK;
}
int32_t mb_timer_stop(mb_ctx* ctx, float* ms_out) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    if (!ms_out) return fail(MB_ERR_INVALID_ARG, "null ms_out");
    MB_CUDA(cudaEventRecord(ctx->ev1, ctx->stream));
    MB_CUDA(cudaEventSynchronize(ctx->ev1));
    MB_CUDA(cudaEventElapsedTime(ms_out, ctx->ev0, ctx->ev1));
    return MB_OK;
}

// ---------------------------------------------------------------------------------- blocks
int32_t mb_block_alloc(mb_ctx* ctx, int32_t rows, int32_t cols, mb_dtype dtype, mb_block** out) {
    if (out) *out = nullptr;
    MB_CTX(ctx);
    if (!out || rows < 0 || cols < 0 || dtype < 0 || dtype > 2) return fail(MB_ERR_INVALID_ARG, "mb_block_alloc: bad argument");
    BlockPtr b(new (std::nothrow) mb_block(), BlockFree{ctx});
    if (!b) return fail(MB_ERR_OOM, "host allocation failed");
    b->rows = rows; b->cols = cols; b->ld = rows > 0 ? rows : 1; b->dtype = dtype; b->owns = 1; b->device = ctx->device;
    const size_t bytes = (size_t)rows * (size_t)cols * elem_size(dtype);
    if (bytes) {
        cudaError_t e = cudaMalloc(&b->data, bytes);
        if (e != cudaSuccess) return cuda_fail(e, "cudaMalloc(block)");
    }
    *out = b.release();
    return MB_OK;
}

int32_t mb_block_wrap(mb_ctx* ctx, void* device_ptr, int64_t offset, int32_t rows, int32_t cols, int32_t ld,
                      int32_t is_transpose, mb_dtype dtype, mb_block** out) {
    if (out) *out = nullptr;
    if (!ctx) return fail(MB_ERR_INVALID_ARG, "null context");
    if (!out || rows < 0 || cols < 0 || offset < 0 || dtype < 0 || dtype > 2)
        return fail(MB_ERR_INVALID_ARG, "mb_block_wrap: bad argument");
    const int minor = is_transpose ? cols : rows;
    if (ld < (minor > 0 ? minor : 1)) return fail(MB_ERR_INVALID_ARG, "mb_block_wrap: ld %d < %d", ld, minor);
    int32_t r = new_block(out);
    if (r) return r;
    mb_block* b = *out;
    b->data = device_ptr; b->offset = offset; b->rows = rows; b->cols = cols; b->ld = ld;
    b->is_transpose = is_transpose ? 1 : 0; b->dtype = dtype; b->owns = 0; b->device = ctx->device;
    return MB_OK;
}

int32_t mb_block_free(mb_ctx* ctx, mb_block* blk) {
    if (!blk) return MB_OK;
    if (blk->owns && blk->data) {
        if (ctx) cudaSetDevice(ctx->device);
        cudaFree(blk->data);
    }
    delete blk;
    return MB_OK;
}

int32_t mb_block_info(const mb_block* blk, int32_t* rows, int32_t* cols, int32_t* ld, int32_t* is_transpose,
                      int32_t* dtype, void** device_ptr) {
    if (!blk) return fail(MB_ERR_INVALID_ARG, "null block");
    if (rows) *rows = blk->rows;
    if (cols) *cols = blk->cols;
    if (ld) *ld = blk->ld;
    if (is_transpose) *is_transpose = blk->is_transpose;
    if (dtype) *dtype = blk->dtype;
    if (device_ptr) *device_ptr = elem_ptr(blk);
    return MB_OK;
}

int32_t mb_block_set_ready_event(mb_block* blk, void* cuda_event) {
    if (!blk) return fail(MB_ERR_INVALID_ARG, "null block");
    blk->ready_event = cuda_event;
    return MB_OK;
}

int32_t mb_block_view_t(mb_ctx* ctx, const mb_block* blk, mb_block** out) {
    if (out) *out = nullptr;
    if (!ctx || !blk || !out) return fail(MB_ERR_INVALID_ARG, "mb_block_view_t: null argument");
    int32_t r = new_block(out);
    if (r) return r;
    **out = transposed(*blk);
    return MB_OK;
}

int32_t mb_block_slice(mb_ctx* ctx, const mb_block* blk, int32_t r0, int32_t r1, int32_t c0, int32_t c1, mb_block** out) {
    if (out) *out = nullptr;
    if (!ctx || !blk || !out) return fail(MB_ERR_INVALID_ARG, "mb_block_slice: null argument");
    if (r0 < 0 || r1 < r0 || r1 > blk->rows || c0 < 0 || c1 < c0 || c1 > blk->cols)
        return fail(MB_ERR_INVALID_ARG, "mb_block_slice: range [%d,%d)x[%d,%d) outside %dx%d", r0, r1, c0, c1, blk->rows, blk->cols);
    int32_t r = new_block(out);
    if (r) return r;
    **out = *blk;
    (*out)->owns = 0;
    (*out)->rows = r1 - r0;
    (*out)->cols = c1 - c0;
    (*out)->offset = blk->offset + r0 * rs(blk) + c0 * cs(blk);
    return MB_OK;
}

int32_t mb_block_upload(mb_ctx* ctx, const double* host, int64_t offset, int32_t rows, int32_t cols, int32_t ld,
                        int32_t is_transpose, mb_dtype store_as, mb_block** out) {
    if (out) *out = nullptr;
    MB_CTX(ctx);
    if (!host || !out || rows < 0 || cols < 0 || offset < 0) return fail(MB_ERR_INVALID_ARG, "mb_block_upload: bad argument");
    const int minor = is_transpose ? cols : rows, major = is_transpose ? rows : cols;
    if (ld < (minor > 0 ? minor : 1)) return fail(MB_ERR_INVALID_ARG, "mb_block_upload: ld %d < %d", ld, minor);
    mb_block* raw = nullptr;
    int32_t r = mb_block_alloc(ctx, rows, cols, store_as, &raw);
    if (r) return r;
    BlockPtr dst(raw, BlockFree{ctx});
    if (rows > 0 && cols > 0) {
        // the raw (minor x major) host array lands in the block, or in a stage one kernel packs / transposes / rounds
        const bool direct = store_as == MB_F64 && !is_transpose;
        mb::StreamBuffer stage;
        if (!direct) MB_CUDA(stage.alloc((size_t)minor * major * 8, ctx->stream));
        MB_CUDA(cudaMemcpy2DAsync(direct ? dst->data : stage.as<void>(), (size_t)minor * 8, host + offset, (size_t)ld * 8,
                                  (size_t)minor * 8, (size_t)major, cudaMemcpyHostToDevice, ctx->stream));
        if (!direct) {
            const mb_block src = block_view(stage.as<void>(), rows, cols, minor, is_transpose, MB_F64, ctx->device);
            r = copy_convert(ctx, &src, dst.get());
        }
        const cudaError_t e = cudaStreamSynchronize(ctx->stream);      // the copy reads the caller's array
        if (r) return r;
        if (e != cudaSuccess) return cuda_fail(e, "mb_block_upload");
    }
    *out = dst.release();
    return MB_OK;
}

int32_t mb_block_download(mb_ctx* ctx, const mb_block* blk, double* host, int32_t ld) {
    MB_CTX(ctx);
    if (!blk || !host) return fail(MB_ERR_INVALID_ARG, "mb_block_download: null argument");
    if (ld < blk->rows) return fail(MB_ERR_INVALID_ARG, "mb_block_download: ld %d < rows %d", ld, blk->rows);
    if (blk->rows == 0 || blk->cols == 0) return MB_OK;
    // fp64 column-major blocks are copied out as they are, others through a packed fp64 copy
    mb_block src = *blk;
    mb::StreamBuffer stage;
    if (blk->dtype != MB_F64 || blk->is_transpose) {
        MB_CUDA(stage.alloc((size_t)blk->rows * blk->cols * 8, ctx->stream));
        src = block_view(stage.as<void>(), blk->rows, blk->cols, blk->rows, false, MB_F64, ctx->device);
        int32_t r = copy_convert(ctx, blk, &src);
        if (r) return r;
    }
    cudaError_t e = cudaMemcpy2DAsync(host, (size_t)ld * 8, f64_ptr(&src), (size_t)src.ld * 8, (size_t)blk->rows * 8,
                                      (size_t)blk->cols, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) return cuda_fail(e, "cudaMemcpy2DAsync(D2H)");
    return MB_OK;
}

// ------------------------------------------------------------------------------------ GEMM
static int32_t dgemm_device_impl(mb_ctx* ctx, char transa, char transb, int32_t m, int32_t n, int32_t k, double alpha,
                                 const double* A, int32_t lda, const double* B, int32_t ldb, double beta, double* C,
                                 int32_t ldc, bool force_generic) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    const bool ta = (transa == 'T' || transa == 't' || transa == 'C' || transa == 'c');
    const bool tb = (transb == 'T' || transb == 't' || transb == 'C' || transb == 'c');
    if (!ta && !(transa == 'N' || transa == 'n')) return fail(MB_ERR_INVALID_ARG, "dgemm: transa '%c'", transa);
    if (!tb && !(transb == 'N' || transb == 'n')) return fail(MB_ERR_INVALID_ARG, "dgemm: transb '%c'", transb);
    if (m < 0 || n < 0 || k < 0) return fail(MB_ERR_INVALID_ARG, "dgemm: negative dimension");
    const int nrowa = ta ? k : m, nrowb = tb ? n : k;
    if (lda < (nrowa > 1 ? nrowa : 1) || ldb < (nrowb > 1 ? nrowb : 1) || ldc < (m > 1 ? m : 1))
        return fail(MB_ERR_INVALID_ARG, "dgemm: leading dimension too small (lda=%d ldb=%d ldc=%d)", lda, ldb, ldc);
    if (m == 0 || n == 0) return MB_OK;
    if (!C || (k > 0 && alpha != 0.0 && (!A || !B))) return fail(MB_ERR_INVALID_ARG, "dgemm: null pointer");
    if (ctx->fp64_mode != MB_FP64_NATIVE && !force_generic && !ta && !tb && alpha == 1.0 && (beta == 0.0 || beta == 1.0) &&
        m >= 256 && n >= 256 && k >= 256 && mb::ozaki_supported(m, n, k, ctx->fp64_slices, ctx->fp64_bits)) {
        cudaError_t e = grow(&ctx->ozaki_ws, &ctx->ozaki_ws_bytes, mb::ozaki_workspace_bytes(m, n, k, ctx->fp64_slices), &ctx->stream);
        if (e != cudaSuccess) return cuda_fail(e, "dgemm: int8-split workspace");
        e = mb::gemm_f64_ozaki(m, n, k, A, lda, B, ldb, C, ldc, beta == 1.0, ctx->fp64_slices, ctx->fp64_bits, ctx->ozaki_ws,
                               ctx->num_sms, ctx->stream);
        if (e == cudaSuccess) return MB_OK;
        if (e != cudaErrorNotSupported) return cuda_fail(e, "gemm_f64_ozaki");
        cudaGetLastError();
    }
    MB_CUDA(mb::gemm_f64(ta, tb, m, n, k, alpha, A, lda, B, ldb, beta, C, ldc, ctx->num_sms, ctx->stream, force_generic));
    return MB_OK;
}

int32_t mb_set_fp64_mode(mb_ctx* ctx, int32_t mode, int32_t slices) {
    if (!ctx) return fail(MB_ERR_INVALID_ARG, "null context");
    if (mode != MB_FP64_NATIVE && mode != MB_FP64_INT8_SPLIT && mode != MB_FP64_INT8_SPLIT8)
        return fail(MB_ERR_INVALID_ARG, "mb_set_fp64_mode: unknown mode %d", mode);
    if (mode != MB_FP64_NATIVE && (slices < 2 || slices > 8)) return fail(MB_ERR_INVALID_ARG, "mb_set_fp64_mode: slices must be in 2..8");
    ctx->fp64_mode = mode;
    if (mode != MB_FP64_NATIVE) { ctx->fp64_slices = slices; ctx->fp64_bits = (mode == MB_FP64_INT8_SPLIT8) ? 8 : 7; }
    return MB_OK;
}

int32_t mb_set_dmma_reference(mb_ctx* ctx, int32_t on) {
    if (!ctx) return fail(MB_ERR_INVALID_ARG, "null context");
    ctx->dmma_reference = on != 0;
    return MB_OK;
}

int32_t mb_dgemm_device(mb_ctx* ctx, char transa, char transb, int32_t m, int32_t n, int32_t k, double alpha,
                        const double* A, int32_t lda, const double* B, int32_t ldb, double beta, double* C, int32_t ldc) {
    return dgemm_device_impl(ctx, transa, transb, m, n, k, alpha, A, lda, B, ldb, beta, C, ldc, false);
}
int32_t mb_dgemm_device_generic(mb_ctx* ctx, char transa, char transb, int32_t m, int32_t n, int32_t k, double alpha,
                                const double* A, int32_t lda, const double* B, int32_t ldb, double beta, double* C,
                                int32_t ldc) {
    return dgemm_device_impl(ctx, transa, transb, m, n, k, alpha, A, lda, B, ldb, beta, C, ldc, true);
}

int32_t mb_dgemm_host(mb_ctx* ctx, char transa, char transb, int32_t m, int32_t n, int32_t k, double alpha,
                      const double* a, int64_t a_offset, int32_t lda, const double* b, int64_t b_offset, int32_t ldb,
                      double beta, double* c, int64_t c_offset, int32_t ldc) {
    MB_CTX(ctx);
    const bool ta = (transa == 'T' || transa == 't'), tb = (transb == 'T' || transb == 't');
    if (m < 0 || n < 0 || k < 0) return fail(MB_ERR_INVALID_ARG, "dgemm: negative dimension");
    if (m == 0 || n == 0) return MB_OK;
    if (!a || !b || !c) return fail(MB_ERR_INVALID_ARG, "dgemm: null host array");
    const int ra = ta ? k : m, ca = ta ? m : k, rb = tb ? n : k, cb = tb ? k : n;
    if (lda < (ra > 1 ? ra : 1) || ldb < (rb > 1 ? rb : 1) || ldc < (m > 1 ? m : 1))
        return fail(MB_ERR_INVALID_ARG, "dgemm: leading dimension too small");
    // device staging is packed with an even leading dimension so the TMA path is always eligible
    auto even = [](int x) { return (x + 1) & ~1; };
    const int dlda = even(ra > 0 ? ra : 1), dldb = even(rb > 0 ? rb : 1), dldc = even(m);
    mb::StreamBuffer bufA, bufB, bufC;
    if (k > 0) {
        MB_CUDA(bufA.alloc((size_t)dlda * ca * 8, ctx->stream));
        MB_CUDA(bufB.alloc((size_t)dldb * cb * 8, ctx->stream));
    }
    MB_CUDA(bufC.alloc((size_t)dldc * n * 8, ctx->stream));
    double *dA = bufA.as<double>(), *dB = bufB.as<double>(), *dC = bufC.as<double>();
    cudaError_t e = cudaSuccess;
    if (k > 0) {
        e = cudaMemcpy2DAsync(dA, (size_t)dlda * 8, a + a_offset, (size_t)lda * 8, (size_t)ra * 8, ca, cudaMemcpyHostToDevice, ctx->stream);
        if (e == cudaSuccess)
            e = cudaMemcpy2DAsync(dB, (size_t)dldb * 8, b + b_offset, (size_t)ldb * 8, (size_t)rb * 8, cb, cudaMemcpyHostToDevice, ctx->stream);
    }
    if (e == cudaSuccess && beta != 0.0)
        e = cudaMemcpy2DAsync(dC, (size_t)dldc * 8, c + c_offset, (size_t)ldc * 8, (size_t)m * 8, n, cudaMemcpyHostToDevice, ctx->stream);
    int32_t r = e == cudaSuccess ? dgemm_device_impl(ctx, transa, transb, m, n, k, alpha, dA, dlda, dB, dldb, beta, dC, dldc, false)
                                 : cuda_fail(e, "H2D copy");
    if (r == MB_OK) {
        e = cudaMemcpy2DAsync(c + c_offset, (size_t)ldc * 8, dC, (size_t)dldc * 8, (size_t)m * 8, n, cudaMemcpyDeviceToHost, ctx->stream);
        if (e != cudaSuccess) r = cuda_fail(e, "D2H copy");
    }
    // the copies read and write the caller's arrays: they have finished when the call returns, whether it failed or not
    e = cudaStreamSynchronize(ctx->stream);
    if (r == MB_OK && e != cudaSuccess) r = cuda_fail(e, "D2H copy");
    return r;
}

// One contraction segment of a bf16 product: op(A) is M x k, op(B) is k x N, stored as the kernel reads them
// (A is M x k if !transA else k x M; B is k x N if !transB else N x k; column-major with leading dimension lda / ldb).
struct bf16_seg {
    const char* a;
    long long lda;
    const char* b;
    long long ldb;
    int k;
};

// The tensor cores add into the fp32 accumulator with truncation, so one accumulation chain drifts in proportion to its
// length in K on same-sign data.  fp32 results are therefore built from chains of at most this many k
// (MARLIN_B200_BF16_KCHAIN, default 8192; 0 = unlimited), read once per process.
static long long bf16_kchain() {
    static const long long v = [] { const char* e = getenv("MARLIN_B200_BF16_KCHAIN"); return e ? atoll(e) : 8192ll; }();
    return v;
}

// C (M x N, column-major, fp32 or bf16) = sum over segs of op(A_s) op(B_s) (+ C if accumulate), for any shape, offset
// and leading dimension:
//   * fp32 C: the segments are cut into chains of at most bf16_kchain() k (and 8 pieces) per launch; the first launch
//     overwrites C unless the caller accumulates, the later ones add into it.  bf16 C: one launch, so one rounding
//     (callers pass at most 8 segments);
//   * a piece whose operand the TMA cannot address (base not 16-byte aligned or ld % 8 != 0: odd block heights,
//     views, cuts inside a segment) is first copied into a packed stream-ordered buffer with ld rounded up to 8.  A
//     copy changes no value, so the result is bit-identical to the same call on aligned operands;
//   * total K = 0 writes zeros into C (nothing under accumulate), as the fp64 path does.
static int32_t bf16_gemm(mb_ctx* ctx, bool ta, bool tb, int M, int N, int nseg, const bf16_seg* segs, void* C,
                         long long ldc, bool c_f32, bool accumulate) {
    if (M <= 0 || N <= 0) return MB_OK;
    const long long cap = (c_f32 && bf16_kchain() > 0) ? bf16_kchain() : (1ll << 62);
    std::vector<bf16_seg> pieces;
    std::vector<size_t> group_end;            // pieces [group_end[g-1], group_end[g]) make launch g
    long long in_group = 0;
    for (int s = 0; s < nseg; ++s)
        for (int k0 = 0; k0 < segs[s].k;) {
            const int len = (int)std::min<long long>(segs[s].k - k0, cap - in_group);
            const bf16_seg& sg = segs[s];
            pieces.push_back({sg.a + 2 * (ta ? (long long)k0 : k0 * sg.lda), sg.lda,     // k0-th row / column of A
                              sg.b + 2 * (tb ? k0 * sg.ldb : (long long)k0), sg.ldb, len});
            in_group += len;
            k0 += len;
            const size_t first = group_end.empty() ? 0 : group_end.back();
            if (in_group >= cap || pieces.size() - first == 8) { group_end.push_back(pieces.size()); in_group = 0; }
        }
    if (group_end.empty() || group_end.back() != pieces.size()) group_end.push_back(pieces.size());
    if (pieces.empty()) {
        if (accumulate) return MB_OK;
        const size_t esz = c_f32 ? 4 : 2;
        MB_CUDA(cudaMemset2DAsync(C, (size_t)ldc * esz, 0, (size_t)M * esz, (size_t)N, ctx->stream));
        return MB_OK;
    }
    auto misaligned = [](const char* p, long long ld) { return (reinterpret_cast<uintptr_t>(p) & 15) != 0 || ld % 8 != 0; };
    std::vector<mb::StreamBuffer> staged;     // the copies of the launch being issued
    // the stored (rows x cols) array of an operand -> a packed copy with ld rounded up to 8 (256-byte aligned base)
    auto stage = [&](const char*& p, long long& ld, int rows, int cols) -> cudaError_t {
        const long long ld8 = (rows + 7) / 8 * 8;
        staged.emplace_back();
        cudaError_t e = staged.back().alloc((size_t)ld8 * cols * 2, ctx->stream);
        if (e != cudaSuccess) return e;
        void* dst = staged.back().as<void>();
        if ((e = mb::convert_strided(MB_BF16, MB_BF16, rows, cols, p, 1, ld, dst, 1, ld8, ctx->stream)) != cudaSuccess) return e;
        p = static_cast<const char*>(dst);
        ld = ld8;
        return cudaSuccess;
    };
    for (size_t g = 0; g < group_end.size(); ++g) {
        const size_t first = g ? group_end[g - 1] : 0;
        const int ns = (int)(group_end[g] - first);
        const void* pa[8]; const void* pb[8]; long long la[8], lb[8]; int ks[8];
        cudaError_t e = cudaSuccess;
        for (int s = 0; s < ns && e == cudaSuccess; ++s) {
            bf16_seg pc = pieces[first + s];
            if (misaligned(pc.a, pc.lda)) e = stage(pc.a, pc.lda, ta ? pc.k : M, ta ? M : pc.k);
            if (e == cudaSuccess && misaligned(pc.b, pc.ldb)) e = stage(pc.b, pc.ldb, tb ? N : pc.k, tb ? pc.k : N);
            pa[s] = pc.a; la[s] = pc.lda; pb[s] = pc.b; lb[s] = pc.ldb; ks[s] = pc.k;
        }
        if (e == cudaSuccess)
            e = mb::gemm_bf16_segments(ta, tb, M, N, ns, ks, pa, la, pb, lb, C, ldc, c_f32, accumulate || g > 0, ctx->num_sms,
                                       ctx->stream);
        staged.clear();
        if (e == cudaErrorNotSupported) return fail(MB_ERR_UNSUPPORTED, "bf16 GEMM: cuTensorMapEncodeTiled is not available");
        if (e != cudaSuccess) return cuda_fail(e, "gemm_bf16_segments");
    }
    return MB_OK;
}

int32_t mb_block_gemm(mb_ctx* ctx, const mb_block* A, const mb_block* B, mb_block* C, int32_t accumulate) {
    MB_CTX(ctx);
    if (!A || !B || !C) return fail(MB_ERR_INVALID_ARG, "mb_block_gemm: null block");
    if (A->cols != B->rows)
        return fail(MB_ERR_DIM_MISMATCH, "Dimension mismatch during matrix-matrix multiplication: %d vs %d", A->cols, B->rows);
    if (C->rows != A->rows || C->cols != B->cols)
        return fail(MB_ERR_DIM_MISMATCH, "mb_block_gemm: result block is %dx%d, expected %dx%d", C->rows, C->cols, A->rows, B->cols);
    const int M = A->rows, N = B->cols, K = A->cols;
    if (A->dtype == MB_F64 && B->dtype == MB_F64 && C->dtype == MB_F64) {
        // degenerate shapes are HBM-bound vector kernels, not tensor-core tiles
        if (N == 1 && M > 1) return mb_block_gemv(ctx, A, B, C, accumulate);                 // matrix x column
        if (M == 1 && N > 1) {                                                              // row x matrix = (B^T a^T)^T
            const mb_block bt = transposed(*B);
            return mb_block_gemv(ctx, &bt, A, C, accumulate);
        }
        if (K == 1 && !accumulate && M > 1 && N > 1) return mb_block_ger(ctx, A, B, C);     // column x row
        if (!C->is_transpose) {
            return dgemm_device_impl(ctx, A->is_transpose ? 'T' : 'N', B->is_transpose ? 'T' : 'N', M, N, K, 1.0, f64_ptr(A),
                                     A->ld, f64_ptr(B), B->ld, accumulate ? 1.0 : 0.0, f64_ptr(C), C->ld, false);
        }
        // row-major result (DenseVecMatrix rows, matrix/DenseVecMatrix.scala:1660-1680): C^T = B^T * A^T,
        // where X^T of a transposed view is the plain column-major array underneath.
        return dgemm_device_impl(ctx, B->is_transpose ? 'N' : 'T', A->is_transpose ? 'N' : 'T', N, M, K, 1.0, f64_ptr(B),
                                 B->ld, f64_ptr(A), A->ld, accumulate ? 1.0 : 0.0, f64_ptr(C), C->ld, false);
    }
    if (A->dtype == MB_BF16 && B->dtype == MB_BF16 && (C->dtype == MB_F32 || C->dtype == MB_BF16)) {
        // any shape, offset and ld (misaligned operands are staged), fp32 chains capped at bf16_kchain()
        if (!C->is_transpose) {
            const bf16_seg seg = {elem_ptr(A), A->ld, elem_ptr(B), B->ld, K};
            return bf16_gemm(ctx, A->is_transpose, B->is_transpose, M, N, 1, &seg, elem_ptr(C), C->ld, C->dtype == MB_F32,
                             accumulate != 0);
        }
        // row-major result: C^T = B^T A^T, as in the fp64 branch
        const bf16_seg seg = {elem_ptr(B), B->ld, elem_ptr(A), A->ld, K};
        return bf16_gemm(ctx, !B->is_transpose, !A->is_transpose, N, M, 1, &seg, elem_ptr(C), C->ld, C->dtype == MB_F32,
                         accumulate != 0);
    }
    return fail(MB_ERR_UNSUPPORTED, "mb_block_gemm: unsupported dtype combination (%d,%d)->%d", A->dtype, B->dtype, C->dtype);
}

// The bytes [lo, hi) a block's elements can occupy.
static void block_span(const mb_block* b, uintptr_t* lo, uintptr_t* hi) {
    const long long major = b->is_transpose ? b->rows : b->cols, minor = b->is_transpose ? b->cols : b->rows;
    *lo = reinterpret_cast<uintptr_t>(elem_ptr(b));
    *hi = *lo + (uintptr_t)(((major - 1) * (long long)b->ld + minor) * (long long)elem_size(b->dtype));
}

// C[e] -= A[e] B[e].  See the header.  Entries whose product mb_block_gemm would run on the DMMA kernel (fp64 native
// mode, M, N, K > 1, column-major C and A, TMA-addressable A and B) become entries of grouped launches with the
// subtracting epilogue; a transposed B is first copied once into a column-major buffer (a copy changes no value).  The
// others run as mb_block_gemm into a temporary and mb_block_sub, which is what the grouped entries reproduce bit for bit.
int32_t mb_block_schur_update(mb_ctx* ctx, int32_t count, mb_block* const* C, const mb_block* const* A,
                              const mb_block* const* B) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    if (count < 0 || (count > 0 && (!C || !A || !B))) return fail(MB_ERR_INVALID_ARG, "mb_block_schur_update: bad argument");
    if (count == 0) return MB_OK;
    std::vector<std::pair<uintptr_t, uintptr_t>> cspan(count);
    for (int e = 0; e < count; ++e) {
        if (!C[e] || !A[e] || !B[e]) return fail(MB_ERR_INVALID_ARG, "mb_block_schur_update: null block in entry %d", e);
        if (C[e]->dtype != MB_F64 || A[e]->dtype != MB_F64 || B[e]->dtype != MB_F64)
            return fail(MB_ERR_UNSUPPORTED, "mb_block_schur_update: fp64 blocks only (entry %d)", e);
        if (A[e]->cols != B[e]->rows || C[e]->rows != A[e]->rows || C[e]->cols != B[e]->cols)
            return fail(MB_ERR_DIM_MISMATCH, "mb_block_schur_update: entry %d is %dx%d -= %dx%d * %dx%d", e, C[e]->rows,
                        C[e]->cols, A[e]->rows, A[e]->cols, B[e]->rows, B[e]->cols);
        if (C[e]->rows == 0 || C[e]->cols == 0) { cspan[e] = {0, 0}; continue; }
        block_span(C[e], &cspan[e].first, &cspan[e].second);
    }
    // no output may overlap another output or any operand: every entry reads what the call was given
    std::vector<std::pair<uintptr_t, uintptr_t>> sorted;
    for (const auto& sp : cspan) if (sp.second > sp.first) sorted.push_back(sp);
    std::sort(sorted.begin(), sorted.end());
    for (size_t x = 1; x < sorted.size(); ++x)
        if (sorted[x].first < sorted[x - 1].second) return fail(MB_ERR_INVALID_ARG, "mb_block_schur_update: two entries share an output");
    auto hits_output = [&](const mb_block* b) {
        if (b->rows == 0 || b->cols == 0) return false;
        uintptr_t lo, hi;
        block_span(b, &lo, &hi);
        auto it = std::lower_bound(sorted.begin(), sorted.end(), std::make_pair(hi, (uintptr_t)0));
        return it != sorted.begin() && std::prev(it)->second > lo;
    };
    for (int e = 0; e < count; ++e)
        if (hits_output(A[e]) || hits_output(B[e]))
            return fail(MB_ERR_INVALID_ARG, "mb_block_schur_update: an operand of entry %d overlaps an output", e);

    const int sms = ctx->num_sms;
    auto grouped = [&](int e) {
        const mb_block *a = A[e], *b = B[e], *c = C[e];
        return ctx->fp64_mode == MB_FP64_NATIVE && a->rows > 1 && a->cols > 1 && b->cols > 1 && !c->is_transpose &&
               !a->is_transpose && mb::gemm_f64_tma_eligible(f64_ptr(a), a->ld, f64_ptr(b), b->ld);
    };
    // column-major copies of the transposed B operands, one per distinct view
    struct Op { const double* p; long long ld; int rows, cols, t; };
    auto same = [](const Op& x, const Op& y) { return x.p == y.p && x.ld == y.ld && x.rows == y.rows && x.cols == y.cols && x.t == y.t; };
    std::vector<Op> copied_of;
    std::vector<mb::StreamBuffer> copies;
    std::vector<Op> bop(count);
    for (int e = 0; e < count; ++e) {
        if (!grouped(e)) continue;
        const mb_block* b = B[e];
        const Op key{f64_ptr(b), b->ld, b->rows, b->cols, b->is_transpose};
        bop[e] = key;
        if (!b->is_transpose) continue;
        size_t x = 0;
        while (x < copied_of.size() && !same(copied_of[x], key)) ++x;
        if (x == copied_of.size()) {
            const int ld = (b->rows + 1) & ~1;
            copies.emplace_back();
            MB_CUDA(copies.back().alloc((size_t)ld * b->cols * sizeof(double), ctx->stream));
            mb_block dst = block_view(copies.back().as<double>(), b->rows, b->cols, ld, false, MB_F64, ctx->device);
            const int32_t r = copy_convert(ctx, b, &dst);
            if (r != MB_OK) return r;
            copied_of.push_back(key);
        }
        bop[e] = Op{copies[x].as<double>(), (b->rows + 1) & ~1, b->rows, b->cols, 0};
    }
    // grouped launches: entries in order, a launch closed when the next entry would exceed its entry or operand limits
    static thread_local mb::G2Launch L;
    L = mb::G2Launch();
    std::vector<Op> la, lb;
    auto flush = [&]() -> cudaError_t {
        const cudaError_t e = mb::gemm_f64_grouped2(L, sms, ctx->stream);
        L = mb::G2Launch();
        la.clear();
        lb.clear();
        return e;
    };
    auto find = [&](const std::vector<Op>& v, const Op& o) {
        for (size_t x = 0; x < v.size(); ++x) if (same(v[x], o)) return (int)x;
        return -1;
    };
    for (int e = 0; e < count; ++e) {
        if (!grouped(e)) continue;
        const Op ao{f64_ptr(A[e]), A[e]->ld, A[e]->rows, A[e]->cols, 0};
        int ia = find(la, ao), ib = find(lb, bop[e]);
        if (L.ne == mb::G2_MAX_ENTRIES || (ia < 0 && L.na == mb::G2_MAX_OPS) || (ib < 0 && L.nb == mb::G2_MAX_OPS)) {
            MB_CUDA(flush());
            ia = ib = -1;
        }
        if (ia < 0) {
            mb::G2Operand& o = L.A[ia = L.na++];
            o.ptr = ao.p; o.ld = ao.ld; o.rows = ao.rows; o.cols = ao.cols;
            la.push_back(ao);
        }
        if (ib < 0) {
            mb::G2Operand& o = L.B[ib = L.nb++];
            o.ptr = bop[e].p; o.ld = bop[e].ld; o.rows = bop[e].rows; o.cols = bop[e].cols;
            lb.push_back(bop[e]);
        }
        mb::G2Entry& en = L.E[L.ne++];
        en.nseg = 1; en.a_op[0] = ia; en.b_op[0] = ib;
        en.M = C[e]->rows; en.N = C[e]->cols;
        en.D = f64_ptr(C[e]); en.ldd = C[e]->ld;
        en.Cin = f64_ptr(C[e]); en.ldcin = C[e]->ld;
        en.sub_from_cin = true;
    }
    if (L.ne > 0) MB_CUDA(flush());
    // the rest: the product into a temporary, then the subtraction in place
    for (int e = 0; e < count; ++e) {
        if (grouped(e) || C[e]->rows == 0 || C[e]->cols == 0) continue;
        const int M = C[e]->rows, N = C[e]->cols;
        mb::StreamBuffer tmp;
        MB_CUDA(tmp.alloc((size_t)M * N * sizeof(double), ctx->stream));
        mb_block t = block_view(tmp.as<double>(), M, N, M, false, MB_F64, ctx->device);
        int32_t r = mb_block_gemm(ctx, A[e], B[e], &t, 0);
        if (r == MB_OK) r = mb_block_sub(ctx, C[e], &t, C[e]);
        if (r != MB_OK) return r;
    }
    return MB_OK;
}

int32_t mb_matmul_blocked_subset(mb_ctx* ctx, mb_block* const* A_tiles, mb_block* const* B_tiles, int32_t m, int32_t k,
                                 int32_t n, mb_block* const* C_tiles, const int32_t* c_ids, int32_t num_c) {
    MB_CTX(ctx);
    if (!A_tiles || !B_tiles || !C_tiles || !c_ids || m <= 0 || k <= 0 || n <= 0 || num_c < 0)
        return fail(MB_ERR_INVALID_ARG, "mb_matmul_blocked: bad argument");
    for (int c = 0; c < num_c; ++c) {
        const int id = c_ids[c];
        if (id < 0 || id >= m * n || !C_tiles[id]) return fail(MB_ERR_INVALID_ARG, "mb_matmul_blocked: bad C id %d", id);
        const int i = id / n, j = id % n;
        for (int kk = 0; kk < k; ++kk) {
            const mb_block *a = A_tiles[i * k + kk], *b = B_tiles[kk * n + j];
            if (!a || !b) return fail(MB_ERR_INVALID_ARG, "mb_matmul_blocked: missing tile for C(%d,%d), kk=%d", i, j, kk);
            if (a->cols != b->rows)
                return fail(MB_ERR_DIM_MISMATCH, "Dimension mismatch during matrix-matrix multiplication: %d vs %d", a->cols, b->rows);
            if (C_tiles[id]->rows != a->rows || C_tiles[id]->cols != b->cols)
                return fail(MB_ERR_DIM_MISMATCH, "mb_matmul_blocked: C(%d,%d) is %dx%d, expected %dx%d", i, j, C_tiles[id]->rows,
                            C_tiles[id]->cols, a->rows, b->cols);
        }
    }
    // ---- grouped single launch when every operand is an fp64 column-major ('N') block ----
    bool groupable = num_c > 0 && ctx->fp64_mode == MB_FP64_NATIVE;
    std::vector<const double*> Ap(m * k, nullptr), Bp(k * n, nullptr);
    std::vector<double*> Cp(m * n, nullptr);
    std::vector<long long> lda(m * k, 2), ldb(k * n, 2), ldc(m * n, 2);
    std::vector<int> row_len(m, -1), k_len(k, -1), col_len(n, -1);    // -1 = not seen yet
    for (int c = 0; c < num_c && groupable; ++c) {
        const int id = c_ids[c], i = id / n, j = id % n;
        const mb_block* cb = C_tiles[id];
        groupable = cb->dtype == MB_F64 && !cb->is_transpose;
        Cp[id] = f64_ptr(cb); ldc[id] = cb->ld;
        for (int kk = 0; kk < k && groupable; ++kk) {
            const mb_block *a = A_tiles[i * k + kk], *b = B_tiles[kk * n + j];
            groupable = a->dtype == MB_F64 && b->dtype == MB_F64 && !a->is_transpose && !b->is_transpose && a->rows > 0 &&
                        a->cols > 0 && b->cols > 0;
            Ap[i * k + kk] = f64_ptr(a); lda[i * k + kk] = a->ld;
            Bp[kk * n + j] = f64_ptr(b); ldb[kk * n + j] = b->ld;
            // the k-slab count is shared by all C blocks: every A(.,kk) must have the same column count
            if (k_len[kk] >= 0 && k_len[kk] != a->cols) groupable = false;
            if (row_len[i] >= 0 && row_len[i] != a->rows) groupable = false;
            if (col_len[j] >= 0 && col_len[j] != b->cols) groupable = false;
            k_len[kk] = a->cols;
            row_len[i] = a->rows; col_len[j] = b->cols;
        }
    }
    if (groupable) {
        cudaError_t e = mb::gemm_f64_grouped(m, k, n, c_ids, num_c, Ap.data(), lda.data(), Bp.data(), ldb.data(), Cp.data(),
                                             ldc.data(), row_len.data(), k_len.data(), col_len.data(), ctx->num_sms, ctx->stream);
        if (e == cudaSuccess) return MB_OK;
        if (e != cudaErrorNotSupported) return cuda_fail(e, "gemm_f64_grouped");
        cudaGetLastError();
    }
    // ---- fallback: seq order of matrix/BlockMatrix.scala:163,168 (p = i*n*k + j*k + kk), the kk partials of C(i,j)
    //      (reduceByKey at :177) accumulated in place, kk ascending ----
    for (int c = 0; c < num_c; ++c) {
        const int id = c_ids[c], i = id / n, j = id % n;
        mb_block* cb = C_tiles[id];
        // bf16 tiles: fold the kk-sum into ONE wgmma launch per C block (K segments; accumulator stays in registers) —
        // per K chain of bf16_kchain() for fp32 C blocks
        bool seg_ok = k <= 8 && !cb->is_transpose && (cb->dtype == MB_F32 || cb->dtype == MB_BF16);
        bf16_seg segs[8];
        for (int kk = 0; kk < k && seg_ok; ++kk) {
            const mb_block *a = A_tiles[i * k + kk], *b = B_tiles[kk * n + j];
            seg_ok = a->dtype == MB_BF16 && b->dtype == MB_BF16 && !a->is_transpose && !b->is_transpose;
            segs[kk] = {elem_ptr(a), a->ld, elem_ptr(b), b->ld, a->cols};
        }
        if (seg_ok) {
            int32_t r = bf16_gemm(ctx, false, false, cb->rows, cb->cols, k, segs, elem_ptr(cb), cb->ld, cb->dtype == MB_F32, false);
            if (r) return r;
            continue;
        }
        for (int kk = 0; kk < k; ++kk) {
            int32_t r = mb_block_gemm(ctx, A_tiles[i * k + kk], B_tiles[kk * n + j], C_tiles[id], kk > 0);
            if (r) return r;
        }
    }
    return MB_OK;
}

int32_t mb_matmul_blocked(mb_ctx* ctx, mb_block* const* A_tiles, mb_block* const* B_tiles, int32_t m, int32_t k,
                          int32_t n, mb_block* const* C_tiles) {
    if (m <= 0 || k <= 0 || n <= 0) return fail(MB_ERR_INVALID_ARG, "mb_matmul_blocked: bad argument");
    std::vector<int32_t> ids(m * n);
    for (int c = 0; c < m * n; ++c) ids[c] = c;
    return mb_matmul_blocked_subset(ctx, A_tiles, B_tiles, m, k, n, C_tiles, ids.data(), m * n);
}

// How mb_matmul_blocked_host cuts one block product so that the tensor cores start before its tiles have crossed PCIe.
// Piece q multiplies k in [k0, k1) of A(i,kk) B(kk,j) into the C columns [c0, c1); it needs only columns [k0, k1) of A
// and that part of B.
//  * along K: the first product, unless it is also the last, when k_len >= 1024 and the tile is non-empty.  The rest of
//    both uploads hides behind the partial products, which accumulate in place.  The cuts are at k_len * q / 4 rounded
//    down to a multiple of 16; the last is k_len.
//  * along the columns: the first and the last product when col_len >= 1024.  The first starts after A and a quarter
//    of B have landed; the last hands each finished column range of C to the D2H stream at once (`download`).
//  * whole: every other product.
struct Piece { int k0, k1, c0, c1; };
struct ProductCut {
    int count = 1;
    Piece piece[4];
    bool along_k = false, download = false;
};
static ProductCut cut_product(bool first, bool last, int rows, int k_len, int cols) {
    ProductCut s;
    s.piece[0] = {0, k_len, 0, cols};
    s.along_k = first && !last && k_len >= 1024 && rows > 0 && cols > 0;
    if (!s.along_k && !((first || last) && cols >= 1024)) return s;
    s.count = 4;
    s.download = last;
    auto kcut = [&](int q) { return q == 4 ? k_len : (int)(((long long)k_len * q / 4) & ~15ll); };
    auto ccut = [&](int q) { return (int)((long long)cols * q / 4); };
    for (int q = 0; q < 4; ++q)
        s.piece[q] = s.along_k ? Piece{kcut(q), kcut(q + 1), 0, cols} : Piece{0, k_len, ccut(q), ccut(q + 1)};
    return s;
}

int32_t mb_matmul_blocked_host(mb_ctx* ctx, const double* const* A_host, const double* const* B_host, int32_t m,
                               int32_t k, int32_t n, const int32_t* row_len, const int32_t* k_len, const int32_t* col_len,
                               double* const* C_host) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    if (!A_host || !B_host || !C_host || !row_len || !k_len || !col_len || m <= 0 || k <= 0 || n <= 0)
        return fail(MB_ERR_INVALID_ARG, "mb_matmul_blocked_host: bad argument");
    MB_CUDA(ensure_copy_streams(ctx));
    ctx->events_used = 0;
    // device layout: every tile gets an even leading dimension and a 256-byte aligned slot (TMA eligibility)
    auto even = [](int x) { return (x + 1) & ~1; };
    auto slot = [](size_t bytes) { return (bytes + 255) & ~size_t(255); };
    std::vector<size_t> offA(m * k), offB(k * n), offC(m * n);
    size_t total = 0;
    for (int i = 0; i < m; ++i)
        for (int kk = 0; kk < k; ++kk) { offA[i * k + kk] = total; total += slot((size_t)even(row_len[i]) * k_len[kk] * 8); }
    for (int kk = 0; kk < k; ++kk)
        for (int j = 0; j < n; ++j) { offB[kk * n + j] = total; total += slot((size_t)even(k_len[kk]) * col_len[j] * 8); }
    for (int i = 0; i < m; ++i)
        for (int j = 0; j < n; ++j) { offC[i * n + j] = total; total += slot((size_t)even(row_len[i]) * col_len[j] * 8); }
    const cudaError_t ge = grow(&ctx->workspace, &ctx->workspace_bytes, total, nullptr);
    if (ge != cudaSuccess) return cuda_fail(ge, "mb_matmul_blocked_host: workspace");
    char* base = static_cast<char*>(ctx->workspace);
    cudaStream_t const S = ctx->stream, h2d = ctx->h2d_stream, d2h = ctx->d2h_stream;
    // `to` waits for everything issued to `from` so far; *at is the event recorded there
    auto handoff = [&](cudaStream_t from, cudaStream_t to, cudaEvent_t* at) {
        cudaError_t e = next_event(ctx, at);
        if (e == cudaSuccess) e = cudaEventRecord(*at, from);
        return e == cudaSuccess ? cudaStreamWaitEvent(to, *at, 0) : e;
    };
    // a rows x cols column-major part of a tile between the host and the workspace (leading dimensions in doubles)
    auto copy = [](double* dst, int dld, const double* src, int sld, int rows, int cols, cudaMemcpyKind kind, cudaStream_t st) {
        if (rows <= 0 || cols <= 0) return cudaSuccess;
        return cudaMemcpy2DAsync(dst, (size_t)dld * 8, src, (size_t)sld * 8, (size_t)rows * 8, cols, kind, st);
    };
    std::vector<cudaEvent_t> evA(m * k, nullptr), evB(k * n, nullptr);     // the tile's upload, once all of it is issued
    // every copy, wait and product of the call in issue order; the first failure ends it
    auto issue = [&]() -> int32_t {
        cudaEvent_t ev = nullptr;
        // the workspace may still be read by a previous call on ctx->stream / d2h_stream: order behind them
        MB_CUDA(handoff(S, h2d, &ev));
        for (int i = 0; i < m; ++i)
            for (int j = 0; j < n; ++j)
                for (int kk = 0; kk < k; ++kk) {
                    const int ia = i * k + kk, ib = kk * n + j, ic = i * n + j;
                    const int rows = row_len[i], depth = k_len[kk], cols = col_len[j];
                    const int lda = std::max(1, even(rows)), ldb = std::max(1, even(depth));     // C has A's leading dimension
                    double *dA = reinterpret_cast<double*>(base + offA[ia]), *dB = reinterpret_cast<double*>(base + offB[ib]),
                           *dC = reinterpret_cast<double*>(base + offC[ic]);
                    const ProductCut cut =
                        cut_product(i == 0 && j == 0 && kk == 0, i == m - 1 && j == n - 1 && kk == k - 1, rows, depth, cols);
                    const bool a_new = !evA[ia], b_new = !evB[ib];
                    for (int q = 0; q < cut.count; ++q) {
                        const Piece& p = cut.piece[q];
                        // uploads in first-use order (seq = i*n*k + j*k + kk); A is cut along K only, B along K or its columns
                        const bool up_a = a_new && (cut.along_k || q == 0);
                        if (up_a)
                            MB_CUDA(copy(dA + (size_t)p.k0 * lda, lda, A_host[ia] + (size_t)p.k0 * rows, rows, rows, p.k1 - p.k0,
                                         cudaMemcpyHostToDevice, h2d));
                        if (b_new)
                            MB_CUDA(copy(dB + (size_t)p.c0 * ldb + p.k0, ldb, B_host[ib] + (size_t)p.c0 * depth + p.k0, depth,
                                         p.k1 - p.k0, p.c1 - p.c0, cudaMemcpyHostToDevice, h2d));
                        // the GEMM waits for this piece's uploads; without any, the first piece waits for the tiles' uploads
                        if (up_a || b_new) {
                            MB_CUDA(handoff(h2d, S, &ev));
                            // a tile whose last part is now issued is complete for the later products
                            if (up_a && p.k1 == depth) evA[ia] = ev;
                            if (b_new && p.k1 == depth && p.c1 == cols) evB[ib] = ev;
                        } else if (q == 0) {
                            MB_CUDA(cudaStreamWaitEvent(S, evA[ia], 0));
                            MB_CUDA(cudaStreamWaitEvent(S, evB[ib], 0));
                        }
                        const int32_t rc = dgemm_device_impl(ctx, 'N', 'N', rows, p.c1 - p.c0, p.k1 - p.k0, 1.0, dA + (size_t)p.k0 * lda,
                                                             lda, dB + (size_t)p.c0 * ldb + p.k0, ldb, (kk > 0 || p.k0 > 0) ? 1.0 : 0.0,
                                                             dC + (size_t)p.c0 * lda, lda, false);
                        if (rc != MB_OK) return rc;
                        if (cut.download) {
                            MB_CUDA(handoff(S, d2h, &ev));
                            MB_CUDA(copy(C_host[ic] + (size_t)p.c0 * rows, rows, dC + (size_t)p.c0 * lda, lda, rows, p.c1 - p.c0,
                                         cudaMemcpyDeviceToHost, d2h));
                        }
                    }
                    // C(i,j) goes to the host after its last kk, unless the last product sent it piece by piece
                    if (kk == k - 1 && !cut.download) {
                        MB_CUDA(handoff(S, d2h, &ev));
                        MB_CUDA(copy(C_host[ic], rows, dC, lda, rows, cols, cudaMemcpyDeviceToHost, d2h));
                    }
                }
        return MB_OK;
    };
    int32_t rc = issue();
    if (rc == MB_OK) {
        // the call returns when every C tile is on the host; ctx->stream is ordered behind the downloads too
        cudaEvent_t ev = nullptr;
        cudaError_t e = handoff(d2h, S, &ev);
        if (e == cudaSuccess) e = cudaStreamSynchronize(d2h);
        if (e != cudaSuccess) rc = cuda_fail(e, "mb_matmul_blocked_host");
    } else {
        cudaStreamSynchronize(h2d); cudaStreamSynchronize(S); cudaStreamSynchronize(d2h);
    }
    return rc;
}

// DenseVecMatrix.multiply(B: BDM) for one row shard (matrix/DenseVecMatrix.scala:1660-1680): C_rows = A_rows * B with
// A_rows / C_rows row-major shards (transposed views) and B the broadcast matrix.
int32_t mb_matmul_rowsharded(mb_ctx* ctx, const mb_block* A_rows, const mb_block* B, mb_block* C_rows) {
    MB_CTX(ctx);
    if (!A_rows || !B || !C_rows) return fail(MB_ERR_INVALID_ARG, "mb_matmul_rowsharded: null block");
    if (A_rows->cols != B->rows)
        return fail(MB_ERR_DIM_MISMATCH, "Dimension mismatch during matrix-matrix multiplication: %d vs %d", A_rows->cols, B->rows);
    return mb_block_gemm(ctx, A_rows, B, C_rows, 0);
}

// The same for JVM-held rows: A_host is the shard's rows back to back (row-major, each row k doubles — exactly the
// `Array[Double]` a partition's rows are packed into at :1672-1675), B_host the column-major k x n broadcast matrix,
// C_host receives the row-major rows x n result.  Row chunks are pipelined: H2D of chunk c+1, the DMMA product of chunk
// c (C^T = B^T * A^T on the row-major data, no transposition pass) and D2H of chunk c-1 run on three streams over a
// ring of three device slots.
int32_t mb_matmul_rowsharded_host(mb_ctx* ctx, const double* A_host, int64_t rows, int32_t k, const double* B_host,
                                  int32_t n, double* C_host) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    if (rows < 0 || k < 0 || n < 0 || (rows > 0 && ((k > 0 && !A_host) || (n > 0 && !C_host))) || (k > 0 && n > 0 && !B_host))
        return fail(MB_ERR_INVALID_ARG, "mb_matmul_rowsharded_host: bad argument");
    if (rows == 0 || n == 0) return MB_OK;
    MB_CUDA(ensure_copy_streams(ctx));
    ctx->events_used = 0;
    constexpr int SLOTS = 3;
    // ~256 MiB of A (or C, whichever is wider) per chunk, a multiple of 128 rows (whole GEMM tiles), at least one tile;
    // MARLIN_B200_ROWSHARD_CHUNK_MIB overrides the size (the tests use it to run many chunks on small inputs)
    long long chunk_mib = 256;
    if (const char* ev = getenv("MARLIN_B200_ROWSHARD_CHUNK_MIB")) chunk_mib = std::max(1, atoi(ev));
    long long chunk = (chunk_mib << 20) / (8ll * std::max(std::max(k, n), 1));
    chunk = std::max(128ll, chunk / 128 * 128);
    chunk = std::min<long long>(chunk, (rows + 127) / 128 * 128);
    const int kk = std::max(k, 1);
    auto slot = [](size_t bytes) { return (bytes + 255) & ~size_t(255); };
    const size_t bytesB = slot((size_t)kk * n * 8), bytesA = slot((size_t)chunk * kk * 8), bytesC = slot((size_t)chunk * n * 8);
    cudaError_t e = grow(&ctx->workspace, &ctx->workspace_bytes, bytesB + SLOTS * (bytesA + bytesC), nullptr);
    if (e != cudaSuccess) return cuda_fail(e, "mb_matmul_rowsharded_host: workspace");
    char* base = static_cast<char*>(ctx->workspace);
    double* dB = reinterpret_cast<double*>(base);
    auto dA = [&](int s_) { return reinterpret_cast<double*>(base + bytesB + (size_t)s_ * (bytesA + bytesC)); };
    auto dC = [&](int s_) { return reinterpret_cast<double*>(base + bytesB + (size_t)s_ * (bytesA + bytesC) + bytesA); };
    cudaEvent_t ev_start = nullptr, ev_b = nullptr, ev_up[SLOTS] = {}, ev_gemm[SLOTS] = {}, ev_down[SLOTS] = {};
    int32_t rc = MB_OK;
    auto mk = [&](cudaEvent_t& ev) { if (e == cudaSuccess) e = next_event(ctx, &ev); };
    mk(ev_start); mk(ev_b);
    for (int s_ = 0; s_ < SLOTS; ++s_) { mk(ev_up[s_]); mk(ev_gemm[s_]); mk(ev_down[s_]); }
    // the workspace may still be in use by an earlier call on ctx->stream
    if (e == cudaSuccess) e = cudaEventRecord(ev_start, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(ctx->h2d_stream, ev_start, 0);
    if (e == cudaSuccess && k > 0) e = cudaMemcpyAsync(dB, B_host, (size_t)k * n * 8, cudaMemcpyHostToDevice, ctx->h2d_stream);
    if (e == cudaSuccess) e = cudaEventRecord(ev_b, ctx->h2d_stream);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(ctx->stream, ev_b, 0);
    const long long nchunks = (rows + chunk - 1) / chunk;
    for (long long c = 0; c < nchunks && e == cudaSuccess && rc == MB_OK; ++c) {
        const int s_ = (int)(c % SLOTS);
        const long long r0 = c * chunk;
        const int nr = (int)std::min<long long>(chunk, rows - r0);
        if (c >= SLOTS) {                       // the slot's previous tenant: its GEMM has read A, its download has read C
            e = cudaStreamWaitEvent(ctx->h2d_stream, ev_gemm[s_], 0);
            if (e == cudaSuccess) e = cudaStreamWaitEvent(ctx->stream, ev_down[s_], 0);
            if (e != cudaSuccess) break;
        }
        if (k > 0) e = cudaMemcpyAsync(dA(s_), A_host + (size_t)r0 * k, (size_t)nr * k * 8, cudaMemcpyHostToDevice, ctx->h2d_stream);
        if (e == cudaSuccess) e = cudaEventRecord(ev_up[s_], ctx->h2d_stream);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(ctx->stream, ev_up[s_], 0);
        if (e != cudaSuccess) break;
        // row-major (nr x n) C chunk == column-major (n x nr) C^T = B^T (n x k) * A^T (k x nr, the row-major chunk itself)
        rc = dgemm_device_impl(ctx, 'T', 'N', n, nr, k, 1.0, dB, kk, dA(s_), kk, 0.0, dC(s_), n, false);
        if (rc != MB_OK) break;
        e = cudaEventRecord(ev_gemm[s_], ctx->stream);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(ctx->d2h_stream, ev_gemm[s_], 0);
        if (e == cudaSuccess) e = cudaMemcpyAsync(C_host + (size_t)r0 * n, dC(s_), (size_t)nr * n * 8, cudaMemcpyDeviceToHost, ctx->d2h_stream);
        if (e == cudaSuccess) e = cudaEventRecord(ev_down[s_], ctx->d2h_stream);
    }
    if (e == cudaSuccess && rc == MB_OK) {
        // returns when every row is on the host; ctx->stream is ordered behind the downloads too
        for (int s_ = 0; s_ < SLOTS && e == cudaSuccess; ++s_)
            if (s_ < nchunks) e = cudaStreamWaitEvent(ctx->stream, ev_down[s_], 0);
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->d2h_stream);
    } else {
        cudaStreamSynchronize(ctx->h2d_stream); cudaStreamSynchronize(ctx->stream); cudaStreamSynchronize(ctx->d2h_stream);
    }
    if (rc != MB_OK) return rc;
    if (e != cudaSuccess) return cuda_fail(e, "mb_matmul_rowsharded_host");
    return MB_OK;
}

// ----------------------------------------------------------------------------- peer memory
int32_t mb_ipc_export(mb_ctx* ctx, const void* device_ptr, uint8_t handle_out[64], int64_t* offset_out, int64_t* alloc_bytes_out) {
    MB_CTX(ctx);
    if (!device_ptr || !handle_out || !offset_out || !alloc_bytes_out) return fail(MB_ERR_INVALID_ARG, "mb_ipc_export: null argument");
    long long off = 0, bytes = 0;
    MB_CUDA(mb::ipc_export(device_ptr, handle_out, &off, &bytes));
    *offset_out = off; *alloc_bytes_out = bytes;
    return MB_OK;
}
int32_t mb_ipc_open(mb_ctx* ctx, const uint8_t handle[64], void** base_out) {
    MB_CTX(ctx);
    if (!handle || !base_out) return fail(MB_ERR_INVALID_ARG, "mb_ipc_open: null argument");
    MB_CUDA(mb::ipc_open(handle, base_out));
    return MB_OK;
}
int32_t mb_ipc_close_all(mb_ctx* ctx) {
    MB_CTX(ctx);
    MB_CUDA(cudaDeviceSynchronize());
    MB_CUDA(mb::ipc_close_all());
    return MB_OK;
}
int32_t mb_flags_alloc(mb_ctx* ctx, int32_t count, void** flags_out) {
    MB_CTX(ctx);
    if (count <= 0 || !flags_out) return fail(MB_ERR_INVALID_ARG, "mb_flags_alloc: bad argument");
    // a private cudaMalloc (not a sub-allocation of somebody's pool), so the exported handle maps exactly this array
    MB_CUDA(cudaMalloc(flags_out, sizeof(unsigned long long) * (size_t)count));
    MB_CUDA(cudaMemset(*flags_out, 0, sizeof(unsigned long long) * (size_t)count));
    MB_CUDA(cudaDeviceSynchronize());
    return MB_OK;
}
int32_t mb_flags_free(mb_ctx* ctx, void* flags) {
    MB_CTX(ctx);
    if (flags) cudaFree(flags);
    return MB_OK;
}
int32_t mb_flag_signal(mb_ctx* ctx, void* flag, int64_t value) {
    MB_CTX(ctx);
    if (!flag) return fail(MB_ERR_INVALID_ARG, "mb_flag_signal: null flag");
    MB_CUDA(mb::flag_signal(flag, (unsigned long long)value, ctx->stream));
    return MB_OK;
}
int32_t mb_flag_wait(mb_ctx* ctx, const void* flag, int64_t value) {
    MB_CTX(ctx);
    if (!flag) return fail(MB_ERR_INVALID_ARG, "mb_flag_wait: null flag");
    MB_CUDA(mb::flag_wait(flag, (unsigned long long)value, ctx->stream));
    return MB_OK;
}
int32_t mb_memcpy_async(mb_ctx* ctx, void* dst, const void* src, int64_t bytes) {
    MB_CTX(ctx);
    if (bytes < 0 || (bytes > 0 && (!dst || !src))) return fail(MB_ERR_INVALID_ARG, "mb_memcpy_async: bad argument");
    if (bytes == 0) return MB_OK;
    MB_CUDA(cudaMemcpyAsync(dst, src, (size_t)bytes, cudaMemcpyDeviceToDevice, ctx->stream));
    return MB_OK;
}

// ----------------------------------------------------------------------------- elementwise
int32_t mb_block_add(mb_ctx* ctx, const mb_block* A, const mb_block* B, mb_block* out) { return binary_op(ctx, mb::EW_ADD, A, B, out, "add"); }
int32_t mb_block_sub(mb_ctx* ctx, const mb_block* A, const mb_block* B, mb_block* out) { return binary_op(ctx, mb::EW_SUB, A, B, out, "subtract"); }
int32_t mb_block_hadamard(mb_ctx* ctx, const mb_block* A, const mb_block* B, mb_block* out) { return binary_op(ctx, mb::EW_MUL, A, B, out, "dotProduct"); }
int32_t mb_block_axpb(mb_ctx* ctx, const mb_block* A, double alpha, double beta, mb_block* out) {
    return unary_op(ctx, mb::EW_AXPB, A, out, alpha, beta, "axpb");
}
int32_t mb_block_fill(mb_ctx* ctx, mb_block* blk, double value) {
    return unary_op(ctx, mb::EW_FILL, blk, blk, 0.0, value, "fill");
}
int32_t mb_block_div(mb_ctx* ctx, const mb_block* A, double b, int32_t b_over_a, mb_block* out) {
    return unary_op(ctx, b_over_a ? mb::EW_RDIV : mb::EW_DIV, A, out, b, 0.0, "divide");
}

int32_t mb_block_copy(mb_ctx* ctx, const mb_block* A, mb_block* out) {
    MB_CTX(ctx);
    if (!A || !out) return fail(MB_ERR_INVALID_ARG, "mb_block_copy: null block");
    int32_t r = same_shape(A, out, "copy");
    if (r) return r;
    return copy_convert(ctx, A, out);
}

int32_t mb_block_transpose(mb_ctx* ctx, const mb_block* A, mb_block* out) {
    MB_CTX(ctx);
    if (!A || !out) return fail(MB_ERR_INVALID_ARG, "mb_block_transpose: null block");
    if (out->rows != A->cols || out->cols != A->rows)
        return fail(MB_ERR_DIM_MISMATCH, "transpose: result block is %dx%d, expected %dx%d", out->rows, out->cols, A->cols, A->rows);
    const mb_block view = transposed(*A);     // A^T as a view, then materialise it (denseBlock.t.copy)
    return copy_convert(ctx, &view, out);
}

int32_t mb_block_sum(mb_ctx* ctx, const mb_block* A, double* sum_out) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    if (!A || !sum_out) return fail(MB_ERR_INVALID_ARG, "mb_block_sum: null argument");
    if (A->dtype != MB_F64) return fail(MB_ERR_UNSUPPORTED, "mb_block_sum: fp64 blocks only");
    if (A->rows == 0 || A->cols == 0) { *sum_out = 0.0; return MB_OK; }
    const int minor = A->is_transpose ? A->cols : A->rows, major = A->is_transpose ? A->rows : A->cols;
    MB_CUDA(mb::sum_f64(f64_ptr(A), minor, major, A->ld, ctx->scratch, ctx->stream));
    MB_CUDA(cudaMemcpyAsync(ctx->host_scalar, ctx->scratch, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    MB_CUDA(cudaStreamSynchronize(ctx->stream));
    *sum_out = *ctx->host_scalar;
    return MB_OK;
}

// DenseVecMatrix.norm (matrix/DenseVecMatrix.scala:975-999) on one row shard: one pass over the view, read in place.
int32_t mb_block_norm(mb_ctx* ctx, const mb_block* A, int32_t kind, mb_block* col_sums, double* out) {
    MB_CTX(ctx);
    if (!A) return fail(MB_ERR_INVALID_ARG, "mb_block_norm: null block");
    if (kind != MB_NORM_ONE && kind != MB_NORM_INF && kind != MB_NORM_FRO)
        return fail(MB_ERR_INVALID_ARG, "mb_block_norm: unknown norm kind %d", kind);
    if (A->dtype != MB_F64) return fail(MB_ERR_UNSUPPORTED, "mb_block_norm: fp64 blocks only");
    vec_view cv{nullptr, 0, 0};
    if (kind == MB_NORM_ONE) {
        if (!col_sums) return fail(MB_ERR_INVALID_ARG, "mb_block_norm: the 1-norm needs a col_sums block");
        if (!as_vector(col_sums, &cv) || cv.len != A->cols)
            return fail(MB_ERR_DIM_MISMATCH, "mb_block_norm: col_sums must be an fp64 vector of %d elements", A->cols);
    } else if (!out) {
        return fail(MB_ERR_INVALID_ARG, "mb_block_norm: null out");
    }
    // RDD.max() of no values; the 1-norm of no columns is the max of no column sums
    if (A->rows == 0 || (kind == MB_NORM_ONE && A->cols == 0)) return fail(MB_ERR_EMPTY, "empty collection");
    if (A->cols == 0) {                                      // rows of no entries: row sums 0.0, no squares
        out[0] = 0.0;
        if (kind == MB_NORM_FRO) out[1] = out[2] = 0.0;
        return MB_OK;
    }
    mb::StreamBuffer ws;
    MB_CUDA(ws.alloc(mb::norm_workspace_bytes(kind, A->rows, A->cols), ctx->stream));
    double* res = nullptr;
    MB_CUDA(mb::norm_f64(kind, f64_ptr(A), rs(A), cs(A), A->rows, A->cols, cv.p, cv.inc, ws.as<void>(), &res, ctx->num_sms,
                         ctx->stream));
    double host[3] = {0.0, 0.0, 0.0};
    const int count = kind == MB_NORM_FRO ? 3 : 1;
    if (out) MB_CUDA(cudaMemcpyAsync(host, res, count * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    MB_CUDA(cudaStreamSynchronize(ctx->stream));
    if (out)
        for (int i = 0; i < count; ++i) out[i] = host[i];
    return MB_OK;
}

int32_t mb_block_gemv(mb_ctx* ctx, const mb_block* A, const mb_block* x, mb_block* y, int32_t accumulate) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    if (!A || !x || !y) return fail(MB_ERR_INVALID_ARG, "mb_block_gemv: null block");
    vec_view xv, yv;
    if (A->dtype != MB_F64 || !as_vector(x, &xv) || !as_vector(y, &yv))
        return fail(MB_ERR_UNSUPPORTED, "mb_block_gemv: fp64 matrix and fp64 single-column (or single-row) vectors only");
    if (A->cols != xv.len)
        return fail(MB_ERR_DIM_MISMATCH, "Dimension mismatch during matrix-vector multiplication: %d vs %d", A->cols, xv.len);
    if (A->rows != yv.len)
        return fail(MB_ERR_DIM_MISMATCH, "mb_block_gemv: result vector has %d elements, expected %d", yv.len, A->rows);
    // a transposed view is the column-major (cols x rows) array underneath: y = S^T x
    const bool trans = A->is_transpose != 0;
    const int m = trans ? A->cols : A->rows, n = trans ? A->rows : A->cols;
    const cudaError_t e = grow(&ctx->vec_ws, &ctx->vec_ws_bytes, mb::gemv_workspace_doubles(trans, m, n) * sizeof(double), &ctx->stream);
    if (e != cudaSuccess) return cuda_fail(e, "mb_block_gemv: workspace");
    MB_CUDA(mb::gemv_f64(trans, m, n, f64_ptr(A), A->ld, xv.p, xv.inc, yv.p, yv.inc, accumulate != 0, ctx->vec_ws, ctx->stream));
    return MB_OK;
}

int32_t mb_block_dot(mb_ctx* ctx, const mb_block* x, const mb_block* y, double* dot_out) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    if (!x || !y || !dot_out) return fail(MB_ERR_INVALID_ARG, "mb_block_dot: null argument");
    vec_view xv, yv;
    if (!as_vector(x, &xv) || !as_vector(y, &yv))
        return fail(MB_ERR_UNSUPPORTED, "mb_block_dot: fp64 single-column (or single-row) vectors only");
    if (xv.len != yv.len)
        return fail(MB_ERR_DIM_MISMATCH, "the length of these two vectors are not the same: %d vs %d", xv.len, yv.len);
    if (xv.len == 0) { *dot_out = 0.0; return MB_OK; }
    MB_CUDA(mb::dot_f64(xv.len, xv.p, xv.inc, yv.p, yv.inc, ctx->scratch, ctx->stream));
    MB_CUDA(cudaMemcpyAsync(ctx->host_scalar, ctx->scratch, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    MB_CUDA(cudaStreamSynchronize(ctx->stream));
    *dot_out = *ctx->host_scalar;
    return MB_OK;
}

int32_t mb_block_ger(mb_ctx* ctx, const mb_block* x, const mb_block* y, mb_block* out) {
    MB_CTX(ctx);
    if (!x || !y || !out) return fail(MB_ERR_INVALID_ARG, "mb_block_ger: null block");
    vec_view xv, yv;
    if (out->dtype != MB_F64 || !as_vector(x, &xv) || !as_vector(y, &yv))
        return fail(MB_ERR_UNSUPPORTED, "mb_block_ger: fp64 vectors and an fp64 result block only");
    if (out->rows != xv.len || out->cols != yv.len)
        return fail(MB_ERR_DIM_MISMATCH, "mb_block_ger: result block is %dx%d, expected %dx%d", out->rows, out->cols, xv.len, yv.len);
    if (out->is_transpose) std::swap(xv, yv);       // (x y^T)^T = y x^T in the array underneath
    MB_CUDA(mb::ger_f64(xv.len, yv.len, xv.p, xv.inc, yv.p, yv.inc, f64_ptr(out), out->ld, ctx->stream));
    return MB_OK;
}

// ---------------------------------------------------------------------- factorizations (SURVEY 8 f4)
static int32_t int_scratch(mb_ctx* ctx, size_t count) {
    const cudaError_t e = grow(&ctx->int_ws, &ctx->int_ws_bytes, count * sizeof(int), &ctx->stream);
    if (e != cudaSuccess) return cuda_fail(e, "factorization workspace");
    if (count > ctx->int_host_count) {
        if (ctx->int_host) { cudaFreeHost(ctx->int_host); ctx->int_host = nullptr; ctx->int_host_count = 0; }
        MB_CUDA(cudaMallocHost(&ctx->int_host, count * sizeof(int)));
        ctx->int_host_count = count;
    }
    return MB_OK;
}
static mb::FView fview(const mb_block* b) { return mb::FView{f64_ptr(b), rs(b), cs(b), b->rows, b->cols}; }

int32_t mb_block_lu(mb_ctx* ctx, mb_block* A, int32_t* perm_out) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    if (!A) return fail(MB_ERR_INVALID_ARG, "mb_block_lu: null block");
    if (A->dtype != MB_F64) return fail(MB_ERR_UNSUPPORTED, "mb_block_lu: fp64 blocks only");
    const int m = A->rows, n = A->cols;
    if (m == 0 || n == 0) return MB_OK;
    int32_t r = int_scratch(ctx, (size_t)2 * m + 8);
    if (r) return r;
    int *piv = ctx->int_ws, *perm = ctx->int_ws + m, *info = ctx->int_ws + 2 * m;
    // rows that are never a pivot position keep themselves: start from the identity interchange
    std::vector<int> ident(m);
    for (int i = 0; i < m; ++i) ident[i] = i;
    std::memcpy(ctx->int_host, ident.data(), sizeof(int) * m);
    MB_CUDA(cudaMemcpyAsync(piv, ctx->int_host, sizeof(int) * m, cudaMemcpyHostToDevice, ctx->stream));
    MB_CUDA(cudaStreamSynchronize(ctx->stream));
    MB_CUDA(mb::getrf(fview(A), piv, nullptr, info, ctx->num_sms, ctx->stream));
    MB_CUDA(cudaMemcpyAsync(ctx->int_host, piv, sizeof(int) * (2 * (size_t)m + 1), cudaMemcpyDeviceToHost, ctx->stream));
    MB_CUDA(cudaStreamSynchronize(ctx->stream));
    if (perm_out) {
        // the reference's pArray (matrix/DenseVecMatrix.scala:303-308): apply the interchanges to 0..m-1
        for (int i = 0; i < m; ++i) perm_out[i] = i;
        for (int i = 0; i < std::min(m, n); ++i) std::swap(perm_out[i], perm_out[ctx->int_host[i]]);
    }
    (void)perm;
    // like Breeze's LU (dgetrf), an exactly singular pivot is not an error here: U carries the zero
    return MB_OK;
}

int32_t mb_block_cholesky(mb_ctx* ctx, mb_block* A) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    if (!A) return fail(MB_ERR_INVALID_ARG, "mb_block_cholesky: null block");
    if (A->dtype != MB_F64) return fail(MB_ERR_UNSUPPORTED, "mb_block_cholesky: fp64 blocks only");
    if (A->rows != A->cols) return fail(MB_ERR_DIM_MISMATCH, "Cholesky needs a square matrix: %d x %d", A->rows, A->cols);
    if (A->rows == 0) return MB_OK;
    int32_t r = int_scratch(ctx, 8);
    if (r) return r;
    MB_CUDA(mb::potrf_lower(fview(A), ctx->int_ws, ctx->num_sms, ctx->stream));
    MB_CUDA(cudaMemcpyAsync(ctx->int_host, ctx->int_ws, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    MB_CUDA(cudaStreamSynchronize(ctx->stream));
    if (ctx->int_host[0] != 0)      // Breeze: NotConvergedException / MatrixNotSymmetricException family -> RuntimeException
        return fail(MB_ERR_CUDA, "Cholesky: the matrix is not positive definite (leading minor %d)", ctx->int_host[0]);
    return MB_OK;
}

int32_t mb_block_inverse(mb_ctx* ctx, const mb_block* A, mb_block* out) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    if (!A || !out) return fail(MB_ERR_INVALID_ARG, "mb_block_inverse: null block");
    if (A->dtype != MB_F64 || out->dtype != MB_F64) return fail(MB_ERR_UNSUPPORTED, "mb_block_inverse: fp64 blocks only");
    if (A->rows != A->cols) return fail(MB_ERR_DIM_MISMATCH, "Inversion only support square matrix: %d v.s %d", A->rows, A->cols);
    if (out->rows != A->rows || out->cols != A->cols) return fail(MB_ERR_DIM_MISMATCH, "mb_block_inverse: result block is %dx%d", out->rows, out->cols);
    const int n = A->rows;
    if (n == 0) return MB_OK;
    int32_t r = int_scratch(ctx, (size_t)2 * n + 8);
    if (r) return r;
    // working copy of A for the factors (packed, even leading dimension)
    const int ld = (n + 1) & ~1;
    mb::StreamBuffer lu;
    MB_CUDA(lu.alloc((size_t)ld * n * sizeof(double), ctx->stream));
    mb_block tmp = block_view(lu.as<void>(), n, n, ld, false, MB_F64, ctx->device);
    r = copy_convert(ctx, A, &tmp);
    if (r) return r;
    int *piv = ctx->int_ws, *info = ctx->int_ws + 2 * n;
    cudaError_t e = mb::getrf(fview(&tmp), piv, nullptr, info, ctx->num_sms, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(ctx->int_host, info, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e == cudaSuccess && ctx->int_host[0] != 0)
        return fail(MB_ERR_CUDA, "matrix is singular (zero pivot in column %d)", ctx->int_host[0] - 1);   // Breeze: MatrixSingularException
    if (e == cudaSuccess) e = mb::inverse_from_lu(fview(&tmp), piv, fview(out), ctx->num_sms, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) return cuda_fail(e, "mb_block_inverse");
    return MB_OK;
}

int32_t mb_block_trsm(mb_ctx* ctx, const mb_block* T, int32_t lower, int32_t unit_diagonal, mb_block* B) {
    MB_CTX(ctx);
    if (!T || !B) return fail(MB_ERR_INVALID_ARG, "mb_block_trsm: null block");
    if (T->dtype != MB_F64 || B->dtype != MB_F64) return fail(MB_ERR_UNSUPPORTED, "mb_block_trsm: fp64 blocks only");
    if (T->rows != T->cols || T->rows != B->rows)
        return fail(MB_ERR_DIM_MISMATCH, "mb_block_trsm: triangle is %dx%d, right-hand side has %d rows", T->rows, T->cols, B->rows);
    MB_CUDA(mb::trsm_left(fview(T), lower != 0, unit_diagonal != 0, fview(B), ctx->num_sms, ctx->stream));
    return MB_OK;
}

// ---------------------------------------------------------------------------------------------------- SVD (SURVEY 8 f5)
// DenseVecMatrix.computeGramianMatrix (matrix/DenseVecMatrix.scala:1464-1486): dspr per row into a packed upper triangle,
// `+=` over partitions, triuToFull.  Here: the lower-triangle tiles on the DMMA mainloop, split over the rows, one
// fixed-order sum of the partials that writes both triangles.
int32_t mb_block_gramian(mb_ctx* ctx, const mb_block* A, mb_block* G) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    if (!A || !G) return fail(MB_ERR_INVALID_ARG, "mb_block_gramian: null block");
    if (A->dtype != MB_F64 || G->dtype != MB_F64) return fail(MB_ERR_UNSUPPORTED, "mb_block_gramian: fp64 blocks only");
    const int m = A->rows, n = A->cols;
    if (n > 65535) return fail(MB_ERR_INVALID_ARG, "Argument with more than 65535 cols: %d", n);
    if (G->rows != n || G->cols != n)
        return fail(MB_ERR_DIM_MISMATCH, "mb_block_gramian: result block is %dx%d, expected %dx%d", G->rows, G->cols, n, n);
    if (n == 0) return MB_OK;
    // a transposed view (a DenseVecMatrix row shard) is the column-major n x m array X underneath: G = X X^T;
    // a column-major view: G = A^T A.  G is symmetric, so a transposed G is written through the same array.
    const bool trans = !A->is_transpose;
    // split-K partials only when the triangle is too small for the SMs (at most 256 MiB), stream-ordered and returned
    // after the call; with one split the product is written into G directly
    const size_t need = mb::gemm_f64_tma_eligible(f64_ptr(A), A->ld, f64_ptr(A), A->ld) ? mb::gram_workspace_doubles(n, m, ctx->num_sms) : 0;
    mb::StreamBuffer ws;
    if (need) MB_CUDA(ws.alloc(need * sizeof(double), ctx->stream));
    const cudaError_t e = mb::gram_f64(trans, n, m, f64_ptr(A), A->ld, f64_ptr(G), G->ld, ws.as<double>(), ctx->num_sms,
                                       ctx->stream);
    if (e != cudaSuccess) return cuda_fail(e, "mb_block_gramian");
    return MB_OK;
}

int64_t mb_gramian_workspace_bytes(int64_t n, int64_t m, int32_t num_sms) {
    if (n <= 0 || n > 65535 || m < 0 || num_sms <= 0) return 0;
    return (int64_t)(mb::gram_workspace_doubles((int)n, m, num_sms) * sizeof(double));
}

// The eigen step of computeSVD (:1589-1606): brzSvd(G) (dgesdd) in local-svd mode, ARPACK's symmetricEigs (:1725-1834) in
// the eigs modes.  One full decomposition by parallel cyclic Jacobi; MB_ERR_NO_CONVERGENCE plays the part of ARPACK's
// IllegalStateException (:1798-1807).
int32_t mb_block_syev(mb_ctx* ctx, const mb_block* G, mb_block* V, double* w_out, int32_t* sweeps_out) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    if (!G || !V || !w_out) return fail(MB_ERR_INVALID_ARG, "mb_block_syev: null argument");
    if (G->dtype != MB_F64 || V->dtype != MB_F64) return fail(MB_ERR_UNSUPPORTED, "mb_block_syev: fp64 blocks only");
    if (G->rows != G->cols) return fail(MB_ERR_DIM_MISMATCH, "mb_block_syev: the matrix is %dx%d, not square", G->rows, G->cols);
    if (V->rows != G->rows || V->cols != G->cols)
        return fail(MB_ERR_DIM_MISMATCH, "mb_block_syev: eigenvector block is %dx%d, expected %dx%d", V->rows, V->cols, G->rows, G->rows);
    constexpr int MAX_SWEEPS = 30;
    int sweeps = 0;
    bool non_finite = false;
    const cudaError_t e = mb::syev_jacobi(G->rows, f64_ptr(G), rs(G), cs(G), f64_ptr(V), rs(V), cs(V), w_out, &sweeps, MAX_SWEEPS,
                                          ctx->stream, &non_finite);
    if (sweeps_out) *sweeps_out = sweeps;
    if (e == cudaSuccess && non_finite)
        return fail(MB_ERR_INVALID_ARG, "mb_block_syev: the matrix holds NaN or Inf (n = %d)", G->rows);
    if (e == cudaErrorNotReady)
        return fail(MB_ERR_NO_CONVERGENCE, "Jacobi eigensolver: no convergence after %d sweeps (n = %d)", MAX_SWEEPS, G->rows);
    if (e != cudaSuccess) return cuda_fail(e, "mb_block_syev");
    return MB_OK;
}

// ------------------------------------------------------------------------------------ logistic regression (DenseVecMatrix.lr)
// The rows of one lr call as the kernel reads them: *v, with row r at f64_ptr(v) + r * rs(v), is A itself when A is a
// row-major view or one column, else a row-major copy in `staged`.  `ws`: n weights, then n gradient values, then the
// per-CTA partials.
static int32_t lr_setup(mb_ctx* ctx, const mb_block* A, const char* name, mb::StreamBuffer* staged, mb::StreamBuffer* ws,
                        mb_block* v) {
    if (!A) return fail(MB_ERR_INVALID_ARG, "%s: null block", name);
    if (A->dtype != MB_F64) return fail(MB_ERR_UNSUPPORTED, "%s: fp64 rows only", name);
    if (A->rows == 0) return fail(MB_ERR_EMPTY, "empty collection");       // numRows() / numCols() on an empty RDD
    if (A->cols == 0) return fail(MB_ERR_INVALID_ARG, "%s: a row needs at least its label (0 columns)", name);
    const int m = A->rows, n = A->cols;
    *v = *A;
    if (!A->is_transpose && n > 1) {
        MB_CUDA(staged->alloc((size_t)m * n * sizeof(double), ctx->stream));
        *v = block_view(staged->as<void>(), m, n, n, true, MB_F64, ctx->device);
        const int32_t r = copy_convert(ctx, A, v);
        if (r) return r;
    }
    MB_CUDA(ws->alloc(((size_t)2 * n + (size_t)mb::lr_parts(m, ctx->num_sms) * n) * sizeof(double), ctx->stream));
    return MB_OK;
}

int32_t mb_lr_gradient(mb_ctx* ctx, const mb_block* rows, const double* w, double* grad) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    if (!w || !grad) return fail(MB_ERR_INVALID_ARG, "mb_lr_gradient: null weights or gradient");
    mb::StreamBuffer staged, ws;
    mb_block v;
    int32_t r = lr_setup(ctx, rows, "mb_lr_gradient", &staged, &ws, &v);
    if (r) return r;
    const int n = v.cols;
    double *wd = ws.as<double>(), *g = wd + n;
    MB_CUDA(cudaMemcpyAsync(wd, w, sizeof(double) * n, cudaMemcpyHostToDevice, ctx->stream));
    MB_CUDA(mb::lr_gradient_f64(f64_ptr(&v), rs(&v), v.rows, n, wd, g + n, g, false, 0.0, ctx->num_sms, ctx->stream));
    MB_CUDA(cudaMemcpyAsync(grad, g, sizeof(double) * n, cudaMemcpyDeviceToHost, ctx->stream));
    MB_CUDA(cudaStreamSynchronize(ctx->stream));
    return MB_OK;
}

int32_t mb_lr_train(mb_ctx* ctx, const mb_block* rows, int64_t data_size, double step, int32_t iters, double* w_out) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    if (!w_out) return fail(MB_ERR_INVALID_ARG, "mb_lr_train: null output");
    if (rows && rows->rows > 0 && data_size <= 0)
        return fail(MB_ERR_INVALID_ARG, "mb_lr_train: data size %lld must be positive", (long long)data_size);
    mb::StreamBuffer staged, ws;
    mb_block v;
    int32_t r = lr_setup(ctx, rows, "mb_lr_train", &staged, &ws, &v);
    if (r) return r;
    const int n = v.cols;
    double* wd = ws.as<double>();
    MB_CUDA(cudaMemsetAsync(wd, 0, sizeof(double) * n, ctx->stream));          // BDV(Array.fill(featureSize)(0.0))
    for (int i = 1; i <= iters; ++i) {
        // weights - delta * (stepSize / dataSize / math.sqrt(i)), the scalar evaluated in that order
        const double scale = step / (double)data_size / std::sqrt((double)i);
        MB_CUDA(mb::lr_gradient_f64(f64_ptr(&v), rs(&v), v.rows, n, wd, wd + 2 * n, nullptr, true, scale, ctx->num_sms,
                                    ctx->stream));
    }
    MB_CUDA(cudaMemcpyAsync(w_out, wd, sizeof(double) * n, cudaMemcpyDeviceToHost, ctx->stream));
    MB_CUDA(cudaStreamSynchronize(ctx->stream));
    return MB_OK;
}

// ------------------------------------------------------------------------ computeSVD dist-eigs: A^T (A x) and Lanczos
// multiplyGramianMatrixBy (matrix/DenseVecMatrix.scala:1444-1459) over one shard.  A row-major view (a row shard's
// transposed view) or a single column is read in place; any other view is first packed into a row-major copy.
int32_t mb_block_gram_matvec(mb_ctx* ctx, const mb_block* A, const mb_block* x, mb_block* y, int32_t accumulate) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    if (!A || !x || !y) return fail(MB_ERR_INVALID_ARG, "mb_block_gram_matvec: null block");
    vec_view xv, yv;
    if (A->dtype != MB_F64 || !as_vector(x, &xv) || !as_vector(y, &yv))
        return fail(MB_ERR_UNSUPPORTED, "mb_block_gram_matvec: fp64 matrix and fp64 single-column (or single-row) vectors only");
    if (A->cols != xv.len)
        return fail(MB_ERR_DIM_MISMATCH, "Dimension mismatch during matrix-vector multiplication: %d vs %d", A->cols, xv.len);
    if (A->cols != yv.len)
        return fail(MB_ERR_DIM_MISMATCH, "mb_block_gram_matvec: result vector has %d elements, expected %d", yv.len, A->cols);
    const int m = A->rows, n = A->cols;
    if (n == 0) return MB_OK;
    mb::StreamBuffer staged, part;
    mb_block v = *A;
    if (!A->is_transpose && n > 1 && m > 0) {
        MB_CUDA(staged.alloc((size_t)m * n * sizeof(double), ctx->stream));
        v = block_view(staged.as<void>(), m, n, n, true, MB_F64, ctx->device);
        const int32_t r = copy_convert(ctx, A, &v);
        if (r) return r;
    }
    const int parts = mb::gram_matvec_parts(m, n, ctx->num_sms);
    if (parts) MB_CUDA(part.alloc((size_t)parts * n * sizeof(double), ctx->stream));
    MB_CUDA(mb::gram_matvec_f64(f64_ptr(&v), rs(&v), m, n, xv.p, xv.inc, yv.p, yv.inc, accumulate != 0, part.as<double>(),
                                ctx->num_sms, ctx->stream));
    return MB_OK;
}

// EigenValueDecomposition.symmetricEigs (:1725-1834) as thick-restart Lanczos (Wu-Simon) with full reorthogonalisation.
// V holds the basis (n x (ncv + 1), column-major) and W the next one while restarting.  The operator writes y = Op x into
// V's next column, which is then orthogonalised in place (classical Gram-Schmidt twice) and normalised.
struct mb_eigs {
    int device = 0;
    int n = 0, nev = 0, ncv = 0;
    double tol = 0.0;
    int32_t max_iter = 0;
    int64_t seed = 0;
    double *V = nullptr, *W = nullptr;   // n x (ncv + 1) each
    double* gemv_ws = nullptr;           // the partial vectors of the basis products
    double* small = nullptr;             // h1, h2, -h (ncv + 1 each), two dot scratches, the ncv x ncv rotation
    double* host = nullptr;              // pinned: h1, h2, |y1|^2, |y2|^2
    mb_block xb, yb;
    std::vector<double> T;               // the projected matrix V^T Op V (ncv x ncv, column-major)
    std::vector<double> w;               // the final eigenvalues (nev, descending) and their vectors in the basis
    std::vector<double> Y;
    int j = -1;                          // Op was asked for V[:, j]; -1 before the start vector
    int iters = 0, draws = 0, nconv = 0;
    int phase = 0;                       // 0 running, 1 converged, 2 out of restarts
    int dot_len = 0;
    double* h1() const { return small; }
    double* h2() const { return small + (ncv + 1); }
    double* hn() const { return small + 2 * (ncv + 1); }
    double* dot1() const { return small + 3 * (ncv + 1); }
    double* dot2() const { return dot1() + dot_len; }
    double* rot() const { return dot2() + dot_len; }
    double* col(double* B, int c) const { return B + (size_t)c * n; }
};

namespace {

constexpr double EIGS_EPS = 0x1p-53;                     // dlamch('EpsMach')
const char* const EIGS_MAX_ITER_MSG =
    "ARPACK returns non-zero info = 1 Maximum number of iterations taken. (Refer ARPACK user guide for details)";

// y := y - V[:, 0:k] (V[:, 0:k]^T y), twice; |y|^2 after each pass into dot1 / dot2 and h of each pass into h1 / h2.
cudaError_t eigs_orthogonalise(mb_ctx* ctx, mb_eigs* E, double* y, int k) {
    const int n = E->n;
    cudaError_t e = cudaSuccess;
    for (int pass = 0; pass < 2 && e == cudaSuccess; ++pass) {
        double* h = pass ? E->h2() : E->h1();
        e = mb::gemv_f64(true, n, k, E->V, n, y, 1, h, 1, false, E->gemv_ws, ctx->stream);
        if (e == cudaSuccess) e = mb::ew_unary(mb::EW_AXPB, k, 1, h, 1, k, E->hn(), 1, k, -1.0, 0.0, ctx->stream);
        if (e == cudaSuccess) e = mb::gemv_f64(false, n, k, E->V, n, E->hn(), 1, y, 1, true, E->gemv_ws, ctx->stream);
        if (e == cudaSuccess) e = mb::dot_f64(n, y, 1, y, 1, pass ? E->dot2() : E->dot1(), ctx->stream);
    }
    return e;
}

// h1, h2 (k each) and the two squared norms to the host: the step's one synchronisation.
cudaError_t eigs_fetch(mb_ctx* ctx, mb_eigs* E, int k) {
    const int c = E->ncv + 1;
    cudaError_t e = cudaMemcpyAsync(E->host, E->h1(), sizeof(double) * k, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(E->host + c, E->h2(), sizeof(double) * k, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(E->host + 2 * c, E->dot1(), sizeof(double), cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(E->host + 2 * c + 1, E->dot2(), sizeof(double), cudaMemcpyDeviceToHost, ctx->stream);
    return e == cudaSuccess ? cudaStreamSynchronize(ctx->stream) : e;
}

// A fresh seeded vector in V[:, k], orthogonal to V[:, 0:k] and normalised (dgetv0).  ARPACK's dgetv0 also gives up
// after a few tries; a vector that survives none of three draws is a failure of the basis, not of the input.
int32_t eigs_fresh(mb_ctx* ctx, mb_eigs* E, int k) {
    const int n = E->n;
    double* v = E->col(E->V, k);
    for (int attempt = 0; attempt < 3; ++attempt) {
        MB_CUDA(mb::fill_uniform_f64(v, 1, n, n, 1, 0, (unsigned long long)mb_hash_seed(E->seed),
                                     (long long)E->draws++ * n, -1.0, 1.0, ctx->stream));
        if (k > 0) {
            MB_CUDA(eigs_orthogonalise(ctx, E, v, k));
        } else {
            MB_CUDA(mb::dot_f64(n, v, 1, v, 1, E->dot2(), ctx->stream));
            MB_CUDA(mb::dot_f64(n, v, 1, v, 1, E->dot1(), ctx->stream));
        }
        MB_CUDA(eigs_fetch(ctx, E, k));
        const double r1 = std::sqrt(E->host[2 * (E->ncv + 1)]), r2 = std::sqrt(E->host[2 * (E->ncv + 1) + 1]);
        if (r2 > 0.717 * r1 && r2 > 0.0) {
            MB_CUDA(mb::ew_unary(mb::EW_DIV, n, 1, v, 1, n, v, 1, n, r2, 0.0, ctx->stream));
            return MB_OK;
        }
    }
    return fail(MB_ERR_NO_CONVERGENCE, "eigs: no start vector independent of the %d-vector basis after three draws", k);
}

// Ask the caller for Op V[:, j], written into V[:, j + 1].
void eigs_request(mb_eigs* E, int32_t* ido, mb_block** x, mb_block** y) {
    E->xb = block_view(E->col(E->V, E->j), E->n, 1, E->n, false, MB_F64, E->device);
    E->yb = block_view(E->col(E->V, E->j + 1), E->n, 1, E->n, false, MB_F64, E->device);
    *x = &E->xb;
    *y = &E->yb;
    *ido = 1;
}

// The basis is full: Ritz pairs of T, the convergence test, and either the end or a thick restart.
int32_t eigs_restart(mb_ctx* ctx, mb_eigs* E, double beta) {
    const int ncv = E->ncv, nev = E->nev, n = E->n;
    std::vector<double> theta(ncv), S((size_t)ncv * ncv);
    int32_t r = mb_eigs_projected(ncv, E->T.data(), theta.data(), S.data());
    if (r) return r;
    // "LM": the wanted pairs are the nev largest in magnitude (ties: larger value first, as sorted)
    std::vector<int> order(ncv);
    for (int i = 0; i < ncv; ++i) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return std::fabs(theta[a]) > std::fabs(theta[b]); });
    const double eps23 = std::pow(EIGS_EPS, 2.0 / 3.0);
    const double floor_res = 0x1p-46 * std::fabs(theta[order[0]]);
    int nconv = 0;
    for (int i = 0; i < nev; ++i) {
        const int c = order[i];
        const double res = std::fabs(beta * S[(size_t)c * ncv + ncv - 1]);
        if (res <= E->tol * std::max(eps23, std::fabs(theta[c])) || res <= floor_res) ++nconv;
    }
    ++E->iters;
    E->nconv = nconv;
    if (nconv >= nev) {
        std::vector<int> want(order.begin(), order.begin() + nev);
        std::stable_sort(want.begin(), want.end(), [&](int a, int b) { return theta[a] > theta[b]; });
        E->w.resize(nev);
        E->Y.resize((size_t)ncv * nev);
        for (int i = 0; i < nev; ++i) {
            E->w[i] = theta[want[i]];
            std::memcpy(E->Y.data() + (size_t)i * ncv, S.data() + (size_t)want[i] * ncv, sizeof(double) * ncv);
        }
        E->phase = 1;
        return MB_OK;
    }
    if (E->iters >= E->max_iter) {
        E->phase = 2;
        return fail(MB_ERR_NO_CONVERGENCE, "%s", EIGS_MAX_ITER_MSG);
    }
    // keep nev + min(nconv, (ncv - nev) / 2) Ritz vectors (dsaup2), at most ncv - 1
    const int kk = std::min(ncv - 1, nev + std::min(nconv, (ncv - nev) / 2));
    std::vector<double> Yk((size_t)ncv * kk);
    for (int i = 0; i < kk; ++i) std::memcpy(Yk.data() + (size_t)i * ncv, S.data() + (size_t)order[i] * ncv, sizeof(double) * ncv);
    MB_CUDA(cudaMemcpyAsync(E->rot(), Yk.data(), sizeof(double) * Yk.size(), cudaMemcpyHostToDevice, ctx->stream));
    mb_block Vb = block_view(E->V, n, ncv, n, false, MB_F64, E->device);
    mb_block Yb = block_view(E->rot(), ncv, kk, ncv, false, MB_F64, E->device);
    mb_block Wb = block_view(E->W, n, kk, n, false, MB_F64, E->device);
    r = mb_block_gemm(ctx, &Vb, &Yb, &Wb, 0);
    if (r) return r;
    MB_CUDA(cudaMemcpyAsync(E->col(E->W, kk), E->col(E->V, ncv), sizeof(double) * n, cudaMemcpyDeviceToDevice, ctx->stream));
    MB_CUDA(cudaStreamSynchronize(ctx->stream));      // Yk leaves scope
    std::swap(E->V, E->W);
    std::fill(E->T.begin(), E->T.end(), 0.0);
    for (int i = 0; i < kk; ++i) {
        E->T[(size_t)i * ncv + i] = theta[order[i]];
        E->T[(size_t)kk * ncv + i] = E->T[(size_t)i * ncv + kk] = beta * S[(size_t)order[i] * ncv + ncv - 1];
    }
    E->j = kk;
    return MB_OK;
}

}  // namespace

int32_t mb_eigs_create(mb_ctx* ctx, int32_t n, int32_t nev, int32_t ncv, double tol, int32_t max_iter, int64_t seed,
                       mb_eigs** out) {
    if (out) *out = nullptr;
    MB_CTX(ctx);
    if (!out) return fail(MB_ERR_INVALID_ARG, "mb_eigs_create: null output");
    if (!(n > nev)) return fail(MB_ERR_INVALID_ARG, "Number of required eigenvalues %d must be smaller than matrix dimension %d", nev, n);
    if (nev <= 0)
        return fail(MB_ERR_INVALID_ARG, "ARPACK returns non-zero info = -2 NEV must be positive. (Refer ARPACK user guide for details)");
    if (!(ncv > nev && ncv <= n))
        return fail(MB_ERR_INVALID_ARG, "ARPACK returns non-zero info = -3 NCV must be greater than NEV and less than or "
                    "equal to N. (Refer ARPACK user guide for details)");
    if (max_iter <= 0)
        return fail(MB_ERR_INVALID_ARG, "ARPACK returns non-zero info = -4 The maximum number of Arnoldi update iterations "
                    "allowed must be greater than zero. (Refer ARPACK user guide for details)");
    std::unique_ptr<mb_eigs, void (*)(mb_eigs*)> E(new (std::nothrow) mb_eigs(), [](mb_eigs* p) { mb_eigs_destroy(p); });
    if (!E) return fail(MB_ERR_OOM, "host allocation failed");
    E->device = ctx->device;
    E->n = n; E->nev = nev; E->ncv = ncv; E->max_iter = max_iter; E->seed = seed;
    E->tol = tol > 0.0 ? tol : EIGS_EPS;
    E->dot_len = mb::dot_scratch_doubles();
    const size_t basis = (size_t)n * (ncv + 1) * sizeof(double);
    const size_t ws = std::max(mb::gemv_workspace_doubles(true, n, ncv + 1), mb::gemv_workspace_doubles(false, n, ncv + 1));
    MB_CUDA(cudaMalloc(&E->V, basis));
    MB_CUDA(cudaMalloc(&E->W, basis));
    MB_CUDA(cudaMalloc(&E->gemv_ws, ws * sizeof(double)));
    MB_CUDA(cudaMalloc(&E->small, (3 * (size_t)(ncv + 1) + 2 * E->dot_len + (size_t)ncv * ncv) * sizeof(double)));
    MB_CUDA(cudaMallocHost(&E->host, (2 * (size_t)(ncv + 1) + 2) * sizeof(double)));
    E->T.assign((size_t)ncv * ncv, 0.0);
    *out = E.release();
    return MB_OK;
}

int32_t mb_eigs_step(mb_ctx* ctx, mb_eigs* E, int32_t* ido, mb_block** x, mb_block** y) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    if (!E || !ido || !x || !y) return fail(MB_ERR_INVALID_ARG, "mb_eigs_step: null argument");
    *x = *y = nullptr;
    if (E->phase == 2) { *ido = 99; return fail(MB_ERR_NO_CONVERGENCE, "%s", EIGS_MAX_ITER_MSG); }
    if (E->phase == 1) { *ido = 99; return MB_OK; }
    const int n = E->n, ncv = E->ncv, c = ncv + 1;
    int32_t r;
    if (E->j < 0) {                                      // the seeded start vector
        r = eigs_fresh(ctx, E, 0);
        if (r) return r;
        E->j = 0;
        eigs_request(E, ido, x, y);
        return MB_OK;
    }
    // the caller wrote Op V[:, j] into V[:, j + 1]
    const int j = E->j, k = j + 1;
    double* v = E->col(E->V, k);
    MB_CUDA(eigs_orthogonalise(ctx, E, v, k));
    MB_CUDA(eigs_fetch(ctx, E, k));
    for (int i = 0; i < k; ++i) {
        const double h = E->host[i] + E->host[c + i];
        E->T[(size_t)j * ncv + i] = E->T[(size_t)i * ncv + j] = h;
    }
    const double r1 = std::sqrt(E->host[2 * c]), r2 = std::sqrt(E->host[2 * c + 1]);
    // the second pass removed much of what the first left: v lies in the basis' span (dsaitr's refinement test)
    const bool invariant = !(r2 > 0.717 * r1) || !(r2 > 0.0);
    double beta = invariant ? 0.0 : r2;
    if (!invariant) {
        MB_CUDA(mb::ew_unary(mb::EW_DIV, n, 1, v, 1, n, v, 1, n, beta, 0.0, ctx->stream));
    } else if (k < ncv) {
        r = eigs_fresh(ctx, E, k);                       // dgetv0: continue from a new direction
        if (r) return r;
    } else {
        MB_CUDA(cudaMemsetAsync(v, 0, sizeof(double) * n, ctx->stream));
    }
    if (k < ncv) {
        E->j = k;
        eigs_request(E, ido, x, y);
        return MB_OK;
    }
    r = eigs_restart(ctx, E, beta);
    if (r) { *ido = 99; return r; }
    if (E->phase == 1) { *ido = 99; return MB_OK; }
    eigs_request(E, ido, x, y);
    return MB_OK;
}

int32_t mb_eigs_result(mb_ctx* ctx, mb_eigs* E, double* w, mb_block* Z, int32_t* nconv, int32_t* iters) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    if (!E) return fail(MB_ERR_INVALID_ARG, "mb_eigs_result: null solver");
    if (nconv) *nconv = E->nconv;
    if (iters) *iters = E->iters;
    if (E->phase == 2) return fail(MB_ERR_NO_CONVERGENCE, "%s", EIGS_MAX_ITER_MSG);
    if (E->phase != 1) return fail(MB_ERR_INVALID_ARG, "mb_eigs_result: the solver has not finished (step until ido = 99)");
    if (w) std::memcpy(w, E->w.data(), sizeof(double) * E->nev);
    if (!Z) return MB_OK;
    if (Z->dtype != MB_F64 || Z->rows != E->n || Z->cols != E->nev)
        return fail(MB_ERR_DIM_MISMATCH, "mb_eigs_result: Z must be an fp64 %d x %d block, got %d x %d", E->n, E->nev, Z->rows, Z->cols);
    MB_CUDA(cudaMemcpyAsync(E->rot(), E->Y.data(), sizeof(double) * E->Y.size(), cudaMemcpyHostToDevice, ctx->stream));
    mb_block Vb = block_view(E->V, E->n, E->ncv, E->n, false, MB_F64, E->device);
    mb_block Yb = block_view(E->rot(), E->ncv, E->nev, E->ncv, false, MB_F64, E->device);
    const int32_t r = mb_block_gemm(ctx, &Vb, &Yb, Z, 0);
    if (r) return r;
    MB_CUDA(cudaStreamSynchronize(ctx->stream));
    return MB_OK;
}

int32_t mb_eigs_destroy(mb_eigs* E) {
    if (!E) return MB_OK;
    int prev = 0;
    cudaGetDevice(&prev);
    cudaSetDevice(E->device);
    cudaDeviceSynchronize();
    cudaFree(E->V);
    cudaFree(E->W);
    cudaFree(E->gemv_ws);
    cudaFree(E->small);
    if (E->host) cudaFreeHost(E->host);
    cudaSetDevice(prev);
    delete E;
    return MB_OK;
}

// ------------------------------------------------------------------------------------------- ALS (CoordinateMatrix.ALS)
// Row i of a row-major fp64 view (a row shard's transposed view, or a single column) at p + i * ld.
static int32_t als_rows(const mb_block* b, const char* what, const double** p, long long* ld) {
    if (!b) return fail(MB_ERR_INVALID_ARG, "ALS: null %s", what);
    if (b->dtype != MB_F64) return fail(MB_ERR_UNSUPPORTED, "ALS: %s must be fp64", what);
    if (!b->is_transpose && b->cols != 1) return fail(MB_ERR_UNSUPPORTED, "ALS: %s must be a row-major view", what);
    *p = f64_ptr(b);
    *ld = b->is_transpose ? b->ld : 1;
    return MB_OK;
}

static int32_t als_check(const mb_als_side* side, int rank, double lambda) {
    if (!side) return fail(MB_ERR_INVALID_ARG, "ALS: null links");
    if (rank < 1) return fail(MB_ERR_INVALID_ARG, "ALS: rank %d must be at least 1", rank);
    if (rank > MB_ALS_MAX_RANK) return fail(MB_ERR_UNSUPPORTED, "ALS: rank %d is above the kernel's cap of %d", rank, MB_ALS_MAX_RANK);
    if (!(lambda >= 0.0)) return fail(MB_ERR_INVALID_ARG, "ALS: lambda %g must be non-negative", lambda);
    if (side->count > 0 && (!side->ids || !side->offsets || !side->partners || !side->ratings || !side->work))
        return fail(MB_ERR_INVALID_ARG, "ALS: null links array");
    return MB_OK;
}

static mb::AlsLinks als_links(const mb_als_side* s) {
    return mb::AlsLinks{s->ids, reinterpret_cast<const long long*>(s->offsets), s->partners, s->ratings, s->work, (long long)s->count};
}

// YtY for implicit mode: the caller's, or the Gramian of Y into `own` (rank x rank)
static int32_t als_yty(mb_ctx* ctx, const mb_block* Yb, const mb_block* YtY, int rank, mb::StreamBuffer* own,
                       const double** p, long long* ld) {
    if (YtY) {
        if (YtY->dtype != MB_F64 || YtY->rows != rank || YtY->cols != rank)
            return fail(MB_ERR_DIM_MISMATCH, "ALS: YtY is %dx%d, expected %dx%d fp64", YtY->rows, YtY->cols, rank, rank);
        *p = f64_ptr(YtY);
        *ld = YtY->ld;          // symmetric: either storage order reads the same element
        return MB_OK;
    }
    MB_CUDA(own->alloc(sizeof(double) * rank * rank, ctx->stream));
    mb_block g = block_view(own->as<void>(), rank, rank, rank, false, MB_F64, ctx->device);
    const int32_t r = mb_block_gramian(ctx, Yb, &g);
    if (r) return r;
    *p = own->as<double>();
    *ld = rank;
    return MB_OK;
}

// One half-step on the ctx stream; *bad (device) collects the lowest failing entity id
static int32_t als_half_step(mb_ctx* ctx, const mb_als_side* side, const mb_block* Yb, double lambda, double alpha,
                             int32_t implicit, const mb_block* YtY, mb_block* Xb, int* bad) {
    const double *Y, *X, *yty = nullptr;
    long long ldy, ldx, ldyty = 0;
    int32_t r = als_rows(Yb, "fixed-side factors", &Y, &ldy);
    if (!r) r = als_rows(Xb, "solved-side factors", &X, &ldx);
    if (r) return r;
    const int rank = Yb->cols;
    if (Xb->cols != rank)
        return fail(MB_ERR_DIM_MISMATCH, "ALS: factors of rank %d and %d", rank, Xb->cols);
    r = als_check(side, rank, lambda);
    if (r) return r;
    mb::StreamBuffer own;
    if (implicit) r = als_yty(ctx, Yb, YtY, rank, &own, &yty, &ldyty);
    if (!r) {
        const cudaError_t e = mb::als_solve(als_links(side), rank, Y, ldy, lambda, alpha, implicit != 0, yty, ldyty,
                                            const_cast<double*>(X), ldx, bad, ctx->stream);
        if (e != cudaSuccess) r = cuda_fail(e, "ALS update");
    }
    return r;
}

// The pivot flag of the half-steps enqueued since it was set to INT32_MAX
static int32_t als_pivots(mb_ctx* ctx, int* bad) {
    MB_CUDA(cudaMemcpyAsync(ctx->int_host, bad, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    MB_CUDA(cudaStreamSynchronize(ctx->stream));
    if (ctx->int_host[0] != INT_MAX)      // Breeze's inv: MatrixSingularException -> RuntimeException
        return fail(MB_ERR_CUDA, "ALS: the normal equations of entity %d are not positive definite", ctx->int_host[0]);
    return MB_OK;
}

static int32_t als_flag(mb_ctx* ctx, int** bad) {
    int32_t r = int_scratch(ctx, 8);
    if (r) return r;
    *bad = ctx->int_ws;
    const int init = INT_MAX;
    MB_CUDA(cudaMemcpyAsync(*bad, &init, sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    MB_CUDA(cudaStreamSynchronize(ctx->stream));          // `init` lives on this frame
    return MB_OK;
}

int32_t mb_als_normal_equations(mb_ctx* ctx, const mb_als_side* side, const mb_block* Yb, double lambda, double alpha,
                                int32_t implicit, const mb_block* YtY, double* A_out, double* b_out) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    const double *Y, *yty = nullptr;
    long long ldy, ldyty = 0;
    int32_t r = als_rows(Yb, "fixed-side factors", &Y, &ldy);
    if (r) return r;
    const int rank = Yb->cols;
    r = als_check(side, rank, lambda);
    if (r) return r;
    if (side->count > 0 && (!A_out || !b_out)) return fail(MB_ERR_INVALID_ARG, "mb_als_normal_equations: null output");
    mb::StreamBuffer own;
    if (implicit) r = als_yty(ctx, Yb, YtY, rank, &own, &yty, &ldyty);
    if (!r) {
        const cudaError_t e = mb::als_assemble(als_links(side), rank, Y, ldy, lambda, alpha, implicit != 0, yty, ldyty, A_out,
                                               b_out, ctx->stream);
        if (e != cudaSuccess) r = cuda_fail(e, "mb_als_normal_equations");
    }
    if (!r) MB_CUDA(cudaStreamSynchronize(ctx->stream));
    return r;
}

int32_t mb_als_update(mb_ctx* ctx, const mb_als_side* side, const mb_block* Y, double lambda, double alpha, int32_t implicit,
                      const mb_block* YtY, mb_block* X) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    int* bad = nullptr;
    int32_t r = als_flag(ctx, &bad);
    if (!r) r = als_half_step(ctx, side, Y, lambda, alpha, implicit, YtY, X, bad);
    return r ? r : als_pivots(ctx, bad);
}

int32_t mb_als_train(mb_ctx* ctx, const mb_als_side* users, const mb_als_side* products, int32_t iterations, double lambda,
                     double alpha, int32_t implicit, mb_block* U, mb_block* P) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    if (!U || !P) return fail(MB_ERR_INVALID_ARG, "mb_als_train: null factors");
    int32_t r = als_check(users, U->cols, lambda);
    if (!r) r = als_check(products, P->cols, lambda);
    if (r || iterations <= 0) return r;
    int* bad = nullptr;
    r = als_flag(ctx, &bad);
    for (int it = 0; it < iterations && !r; ++it) {
        r = als_half_step(ctx, products, U, lambda, alpha, implicit, nullptr, P, bad);      // products from the users
        if (!r) r = als_half_step(ctx, users, P, lambda, alpha, implicit, nullptr, U, bad); // then users from the products
    }
    return r ? r : als_pivots(ctx, bad);
}

int32_t mb_als_update_host(mb_ctx* ctx, int32_t rank, int64_t n_fixed, const double* Y, int64_t n, const int64_t* ids,
                           const int64_t* offsets, const int32_t* partners, const float* ratings, double lambda,
                           double alpha, int32_t implicit, const double* YtY, double* X) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    if (n < 0 || n_fixed < 0 || (n > 0 && (!ids || !offsets || !X)) || (n_fixed > 0 && !Y) || (n > 0 && offsets[n] > 0 && (!partners || !ratings)))
        return fail(MB_ERR_INVALID_ARG, "mb_als_update_host: bad argument");
    if (n == 0) return MB_OK;
    const mb_als_side none{};
    int32_t r = als_check(&none, rank, lambda);
    if (r) return r;
    if (n > INT32_MAX) return fail(MB_ERR_UNSUPPORTED, "mb_als_update_host: %lld entities", (long long)n);
    if (offsets[0] != 0) return fail(MB_ERR_INVALID_ARG, "mb_als_update_host: offsets[0] is %lld, not 0", (long long)offsets[0]);
    for (int64_t p = 0; p < n; ++p)
        if (offsets[p + 1] < offsets[p])
            return fail(MB_ERR_INVALID_ARG, "mb_als_update_host: offsets decrease at entity %lld", (long long)p);
    const int64_t nnz = offsets[n];
    for (int64_t q = 0; q < nnz; ++q)
        if (partners[q] < 0 || partners[q] >= n_fixed)
            return fail(MB_ERR_INVALID_ARG, "mb_als_update_host: partner %d outside the %lld fixed rows", partners[q], (long long)n_fixed);
    std::vector<int32_t> ids32(n), work(n);
    for (int64_t p = 0; p < n; ++p) {
        if (ids[p] < 0 || ids[p] > INT32_MAX) return fail(MB_ERR_INVALID_ARG, "ALS: id %lld is outside [0, 2147483647]", (long long)ids[p]);
        ids32[p] = int32_t(ids[p]);
        work[p] = int32_t(p);
    }
    std::stable_sort(work.begin(), work.end(), [&](int32_t a, int32_t b) { return offsets[a + 1] - offsets[a] > offsets[b + 1] - offsets[b]; });
    mb::StreamBuffer d_ids, d_off, d_partners, d_r, d_work, d_y, d_x, d_yty;
    MB_CUDA(d_ids.upload(ids32.data(), sizeof(int32_t) * n, ctx->stream));
    MB_CUDA(d_off.upload(offsets, sizeof(int64_t) * (n + 1), ctx->stream));
    MB_CUDA(d_partners.upload(partners, sizeof(int32_t) * nnz, ctx->stream));
    MB_CUDA(d_r.upload(ratings, sizeof(float) * nnz, ctx->stream));
    MB_CUDA(d_work.upload(work.data(), sizeof(int32_t) * n, ctx->stream));
    MB_CUDA(d_y.upload(Y, sizeof(double) * n_fixed * rank, ctx->stream));
    MB_CUDA(d_x.upload(X, sizeof(double) * n * rank, ctx->stream));
    if (YtY) MB_CUDA(d_yty.upload(YtY, sizeof(double) * rank * rank, ctx->stream));
    const mb_als_side side{n, d_ids.as<int32_t>(), d_off.as<int64_t>(), d_partners.as<int32_t>(), d_r.as<float>(),
                           d_work.as<int32_t>()};
    const mb_block yb = block_view(d_y.as<void>(), (int)n_fixed, rank, rank, true, MB_F64, ctx->device);
    const mb_block gb = block_view(d_yty.as<void>(), rank, rank, rank, true, MB_F64, ctx->device);
    mb_block xb = block_view(d_x.as<void>(), (int)n, rank, rank, true, MB_F64, ctx->device);
    r = mb_als_update(ctx, &side, &yb, lambda, alpha, implicit, YtY ? &gb : nullptr, &xb);
    if (r) return r;
    MB_CUDA(cudaMemcpyAsync(X, d_x.as<void>(), sizeof(double) * n * rank, cudaMemcpyDeviceToHost, ctx->stream));
    MB_CUDA(cudaStreamSynchronize(ctx->stream));
    return MB_OK;
}

int32_t mb_coo_to_dense_rows(mb_ctx* ctx, int64_t nnz, const int32_t* row_pos, const int32_t* cols, const float* values,
                             mb_block* out) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    const double* p;
    long long ld;
    int32_t r = als_rows(out, "toDenseVecMatrix output", &p, &ld);
    if (r) return r;
    if (nnz < 0 || (nnz > 0 && (!row_pos || !cols || !values))) return fail(MB_ERR_INVALID_ARG, "mb_coo_to_dense_rows: bad argument");
    std::vector<int64_t> keys((size_t)nnz);
    for (int64_t e = 0; e < nnz; ++e) {
        if (row_pos[e] < 0 || row_pos[e] >= out->rows || cols[e] < 0 || cols[e] >= out->cols)
            return fail(MB_ERR_INVALID_ARG, "toDenseVecMatrix: entry (%d, %d) is outside the %dx%d rows", row_pos[e], cols[e],
                        out->rows, out->cols);
        keys[e] = (int64_t)row_pos[e] * out->cols + cols[e];
    }
    std::sort(keys.begin(), keys.end());
    for (size_t e = 1; e < keys.size(); ++e)      // Vectors.sparse (matrix/Vectors.scala:92-104)
        if (keys[e] == keys[e - 1])
            return fail(MB_ERR_INVALID_ARG, "requirement failed: Found duplicate indices: %lld.", (long long)(keys[e] % out->cols));
    if (ld == out->cols || out->rows == 1)
        MB_CUDA(cudaMemsetAsync(const_cast<double*>(p), 0, sizeof(double) * out->rows * out->cols, ctx->stream));
    else
        MB_CUDA(cudaMemset2DAsync(const_cast<double*>(p), sizeof(double) * ld, 0, sizeof(double) * out->cols, out->rows, ctx->stream));
    mb::StreamBuffer d_row, d_col, d_val;
    MB_CUDA(d_row.upload(row_pos, sizeof(int32_t) * nnz, ctx->stream));
    MB_CUDA(d_col.upload(cols, sizeof(int32_t) * nnz, ctx->stream));
    MB_CUDA(d_val.upload(values, sizeof(float) * nnz, ctx->stream));
    MB_CUDA(mb::coo_scatter_rows(nnz, d_row.as<int32_t>(), d_col.as<int32_t>(), d_val.as<float>(), const_cast<double*>(p), ld,
                                 ctx->stream));
    MB_CUDA(cudaStreamSynchronize(ctx->stream));
    return MB_OK;
}

int32_t mb_fill_uniform(mb_ctx* ctx, mb_block* blk, int64_t partition_seed, int64_t first, double lo, double hi,
                        int32_t row_major) {
    MB_CTX(ctx);
    if (!blk || first < 0) return fail(MB_ERR_INVALID_ARG, "mb_fill_uniform: bad argument");
    if (blk->dtype != MB_F64) return fail(MB_ERR_UNSUPPORTED, "mb_fill_uniform: fp64 blocks only (convert afterwards)");
    // generator.setSeed(partition.seed) -> XORShiftRandom.setSeed -> seed = hashSeed(s)
    const unsigned long long state0 = (unsigned long long)mb_hash_seed(partition_seed);
    MB_CUDA(mb::fill_uniform_f64(f64_ptr(blk), rs(blk), cs(blk), blk->rows, blk->cols, row_major ? 1 : 0, state0, first, lo,
                                 hi, ctx->stream));
    return MB_OK;
}

static_assert(MB_NORMAL_TILE_ATTEMPTS == mb::NORMAL_TILE_ATTEMPTS, "the documented tile size is the kernels' tile size");

// generator.setSeed(partition.seed) and Array.fill(n)(nextValue()) of StandardNormalGenerator into an fp64 view; the counted
// attempts may reach `extra` positions short of the jump tables' 2^39 (room for what the caller draws after the values)
static int32_t fill_normal(mb_ctx* ctx, double* out, long long rs, long long cs, int rows, int cols, int row_major,
                           int64_t partition_seed, double mean, double variance, long long extra, int64_t* positions,
                           const char* what) {
    const unsigned long long state0 = (unsigned long long)mb_hash_seed(partition_seed);
    long long attempts = 0;
    const cudaError_t e = mb::fill_normal_f64(out, rs, cs, rows, cols, row_major, state0, mean, std::sqrt(variance),
                                              (1LL << 39) - 1 - extra, positions ? &attempts : nullptr, ctx->stream);
    if (e == cudaErrorInvalidValue)
        return fail(MB_ERR_UNSUPPORTED, "%s: %dx%d values exceed the generator's 2^39 stream positions", what, rows, cols);
    if (e != cudaSuccess) return cuda_fail(e, what);
    if (positions) *positions = 2 * attempts;
    return MB_OK;
}

int32_t mb_fill_normal(mb_ctx* ctx, mb_block* blk, int64_t partition_seed, double mean, double variance, int32_t row_major,
                       int64_t* positions_out) {
    MB_CTX(ctx);
    if (positions_out) *positions_out = 0;
    if (!blk) return fail(MB_ERR_INVALID_ARG, "mb_fill_normal: bad argument");
    if (blk->dtype != MB_F64) return fail(MB_ERR_UNSUPPORTED, "mb_fill_normal: fp64 blocks only (convert afterwards)");
    return fill_normal(ctx, f64_ptr(blk), rs(blk), cs(blk), blk->rows, blk->cols, row_major ? 1 : 0, partition_seed, mean,
                       variance, 0, positions_out, "mb_fill_normal");
}

// ------------------------------------------------------------------------------------------- sparse blocks (SURVEY 8 f6)
static mb::CscView csc(const mb_sparse* S) { return mb::CscView{S->rows, S->cols, S->colptr, S->rowidx, S->values}; }
static mb::DView dview(const mb_block* b) { return mb::DView{f64_ptr(b), rs(b), cs(b)}; }

int32_t mb_sparse_wrap(mb_ctx* ctx, int32_t rows, int32_t cols, int64_t nnz, void* colptr, void* rowidx, void* values,
                       mb_sparse** out) {
    if (out) *out = nullptr;
    if (!ctx) return fail(MB_ERR_INVALID_ARG, "null context");
    if (!out || rows < 0 || cols < 0 || nnz < 0 || !colptr || (nnz > 0 && (!rowidx || !values)))
        return fail(MB_ERR_INVALID_ARG, "mb_sparse_wrap: bad argument");
    if (nnz > 0x7fffffffLL) return fail(MB_ERR_INVALID_ARG, "sparse block with %lld non-zeros: at most 2^31 - 1", (long long)nnz);
    mb_sparse* S = new (std::nothrow) mb_sparse();
    if (!S) return fail(MB_ERR_OOM, "host allocation failed");
    S->rows = rows; S->cols = cols; S->nnz = nnz; S->device = ctx->device;
    S->colptr = static_cast<int*>(colptr); S->rowidx = static_cast<int*>(rowidx); S->values = static_cast<double*>(values);
    *out = S;
    return MB_OK;
}

int32_t mb_sparse_upload(mb_ctx* ctx, int32_t rows, int32_t cols, const int32_t* colptr, const int32_t* rowidx,
                         const double* values, mb_sparse** out) {
    if (out) *out = nullptr;
    MB_CTX(ctx);
    if (!out || !colptr) return fail(MB_ERR_INVALID_ARG, "mb_sparse_upload: null argument");
    int32_t r = mb_sparse_check(rows, cols, colptr, rowidx);
    if (r) return r;
    const long long nnz = colptr[cols];
    if (nnz > 0 && !values) return fail(MB_ERR_INVALID_ARG, "mb_sparse_upload: null values");
    mb_sparse* raw = nullptr;
    if ((r = mb_sparse_alloc(ctx, rows, cols, nnz, &raw)) != MB_OK) return r;
    SparsePtr S(raw, SparseFree{ctx});
    cudaError_t e = cudaMemcpy(S->colptr, colptr, sizeof(int) * ((size_t)cols + 1), cudaMemcpyHostToDevice);
    if (e == cudaSuccess && nnz) e = cudaMemcpy(S->rowidx, rowidx, sizeof(int) * (size_t)nnz, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && nnz) e = cudaMemcpy(S->values, values, sizeof(double) * (size_t)nnz, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) return cuda_fail(e, "mb_sparse_upload");
    *out = S.release();
    return MB_OK;
}

int32_t mb_sparse_download(mb_ctx* ctx, const mb_sparse* S, int32_t* colptr, int32_t* rowidx, double* values) {
    MB_CTX(ctx);
    if (!S || !colptr || (S->nnz > 0 && (!rowidx || !values))) return fail(MB_ERR_INVALID_ARG, "mb_sparse_download: null argument");
    MB_CUDA(cudaStreamSynchronize(ctx->stream));
    MB_CUDA(cudaMemcpy(colptr, S->colptr, sizeof(int) * ((size_t)S->cols + 1), cudaMemcpyDeviceToHost));
    if (S->nnz) {
        MB_CUDA(cudaMemcpy(rowidx, S->rowidx, sizeof(int) * (size_t)S->nnz, cudaMemcpyDeviceToHost));
        MB_CUDA(cudaMemcpy(values, S->values, sizeof(double) * (size_t)S->nnz, cudaMemcpyDeviceToHost));
    }
    return MB_OK;
}

int32_t mb_sparse_info(const mb_sparse* S, int32_t* rows, int32_t* cols, int64_t* nnz) {
    if (!S) return fail(MB_ERR_INVALID_ARG, "null sparse block");
    if (rows) *rows = S->rows;
    if (cols) *cols = S->cols;
    if (nnz) *nnz = S->nnz;
    return MB_OK;
}

int32_t mb_sparse_alloc(mb_ctx* ctx, int32_t rows, int32_t cols, int64_t nnz, mb_sparse** out) {
    if (out) *out = nullptr;
    MB_CTX(ctx);
    if (!out || rows < 0 || cols < 0 || nnz < 0) return fail(MB_ERR_INVALID_ARG, "mb_sparse_alloc: bad argument");
    if (nnz > 0x7fffffffLL) return fail(MB_ERR_INVALID_ARG, "sparse block with %lld non-zeros: at most 2^31 - 1", (long long)nnz);
    SparsePtr S(new (std::nothrow) mb_sparse(), SparseFree{ctx});
    if (!S) return fail(MB_ERR_OOM, "host allocation failed");
    S->rows = rows; S->cols = cols; S->nnz = nnz; S->owns = 1; S->device = ctx->device;
    cudaError_t e = cudaMalloc(&S->colptr, sizeof(int) * ((size_t)cols + 1));
    if (e == cudaSuccess && nnz) e = cudaMalloc(&S->rowidx, sizeof(int) * (size_t)nnz);
    if (e == cudaSuccess && nnz) e = cudaMalloc(&S->values, sizeof(double) * (size_t)nnz);
    if (e != cudaSuccess) return cuda_fail(e, "mb_sparse_alloc");
    *out = S.release();
    return MB_OK;
}

int32_t mb_sparse_values_op(mb_ctx* ctx, const mb_sparse* S, int32_t op, double b, mb_sparse** out) {
    if (out) *out = nullptr;
    MB_CTX(ctx);
    if (!S || !out || op < MB_SPARSE_ADD || op > MB_SPARSE_DIV) return fail(MB_ERR_INVALID_ARG, "mb_sparse_values_op: bad argument");
    mb_sparse* raw = nullptr;
    int32_t r = mb_sparse_alloc(ctx, S->rows, S->cols, S->nnz, &raw);
    if (r) return r;
    SparsePtr R(raw, SparseFree{ctx});
    cudaError_t e = cudaMemcpyAsync(R->colptr, S->colptr, sizeof(int) * ((size_t)S->cols + 1), cudaMemcpyDeviceToDevice, ctx->stream);
    if (e == cudaSuccess && S->nnz)
        e = cudaMemcpyAsync(R->rowidx, S->rowidx, sizeof(int) * (size_t)S->nnz, cudaMemcpyDeviceToDevice, ctx->stream);
    if (e == cudaSuccess && S->nnz) {
        // the values as an nnz x 1 block through the dense kernels: the same arithmetic as SubMatrix.add(b) etc. on a dense block
        const int n = (int)S->nnz;
        if (op == MB_SPARSE_DIV) e = mb::ew_unary(mb::EW_DIV, n, 1, S->values, 1, n, R->values, 1, n, b, 0.0, ctx->stream);
        else {
            const double alpha = op == MB_SPARSE_MUL ? b : 1.0;
            const double beta = op == MB_SPARSE_ADD ? b : (op == MB_SPARSE_SUB ? -b : 0.0);
            e = mb::ew_unary(mb::EW_AXPB, n, 1, S->values, 1, n, R->values, 1, n, alpha, beta, ctx->stream);
        }
    }
    if (e != cudaSuccess) return cuda_fail(e, "mb_sparse_values_op");
    *out = R.release();
    return MB_OK;
}

int32_t mb_sparse_free(mb_ctx* ctx, mb_sparse* S) {
    if (!S) return MB_OK;
    if (ctx) {
        cudaSetDevice(ctx->device);
        cudaStreamSynchronize(ctx->stream);      // a product may still read the CSR copy
    }
    if (S->owns) {
        cudaFree(S->colptr);
        cudaFree(S->rowidx);
        cudaFree(S->values);
    }
    cudaFree(S->csr_rowptr);
    cudaFree(S->csr_colidx);
    cudaFree(S->csr_values);
    cudaFree(S->pagerank_heavy);
    delete S;
    return MB_OK;
}

static int32_t dense_f64_out(const mb_block* C, int rows, int cols, const char* what) {
    if (C->dtype != MB_F64) return fail(MB_ERR_UNSUPPORTED, "%s: fp64 blocks only", what);
    if (C->rows != rows || C->cols != cols)
        return fail(MB_ERR_DIM_MISMATCH, "%s: result block is %dx%d, expected %dx%d", what, C->rows, C->cols, rows, cols);
    return MB_OK;
}

int32_t mb_sparse_to_dense(mb_ctx* ctx, const mb_sparse* S, mb_block* out) {
    MB_CTX(ctx);
    if (!S || !out) return fail(MB_ERR_INVALID_ARG, "mb_sparse_to_dense: null argument");
    int32_t r = dense_f64_out(out, S->rows, S->cols, "toDense");
    if (r) return r;
    MB_CUDA(mb::csc_to_dense(csc(S), dview(out), ctx->stream));
    return MB_OK;
}

int32_t mb_spmm_dense_sparse(mb_ctx* ctx, const mb_block* A, const mb_sparse* B, mb_block* C, int32_t accumulate) {
    MB_CTX(ctx);
    if (!A || !B || !C) return fail(MB_ERR_INVALID_ARG, "mb_spmm_dense_sparse: null argument");
    if (A->dtype != MB_F64) return fail(MB_ERR_UNSUPPORTED, "multDenseSparse: fp64 blocks only");
    if (A->cols != B->rows) return fail(MB_ERR_DIM_MISMATCH, "matrix dimension mismatch: %d v.s %d", A->cols, B->rows);
    int32_t r = dense_f64_out(C, A->rows, B->cols, "multDenseSparse");
    if (r) return r;
    MB_CUDA(mb::spmm_dense_sparse(A->rows, dview(A), csc(B), dview(C), accumulate != 0, ctx->stream));
    return MB_OK;
}

int32_t mb_spmm_sparse_dense(mb_ctx* ctx, mb_sparse* A, const mb_block* B, mb_block* C, int32_t accumulate) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    if (!A || !B || !C) return fail(MB_ERR_INVALID_ARG, "mb_spmm_sparse_dense: null argument");
    if (B->dtype != MB_F64) return fail(MB_ERR_UNSUPPORTED, "multSparseDense: fp64 blocks only");
    if (A->cols != B->rows) return fail(MB_ERR_DIM_MISMATCH, "matrix dimension mismatch: %d v.s %d", A->cols, B->rows);
    int32_t r = dense_f64_out(C, A->rows, B->cols, "multSparseDense");
    if (r) return r;
    if (!A->csr_rowptr) {
        int *rowptr = nullptr, *colidx = nullptr;
        double* vals = nullptr;
        cudaError_t e = cudaMalloc(&rowptr, sizeof(int) * ((size_t)A->rows + 1));
        if (e == cudaSuccess) e = cudaMalloc(&colidx, sizeof(int) * std::max<size_t>(1, (size_t)A->nnz));
        if (e == cudaSuccess) e = cudaMalloc(&vals, sizeof(double) * std::max<size_t>(1, (size_t)A->nnz));
        if (e == cudaSuccess) e = mb::csc_to_csr(csc(A), A->nnz, rowptr, colidx, vals, ctx->stream);
        if (e != cudaSuccess) {
            cudaFree(rowptr); cudaFree(colidx); cudaFree(vals);
            return cuda_fail(e, "multSparseDense: CSR copy");
        }
        A->csr_rowptr = rowptr; A->csr_colidx = colidx; A->csr_values = vals;
    }
    const mb::CsrView csr{A->rows, A->cols, A->csr_rowptr, A->csr_colidx, A->csr_values};
    MB_CUDA(mb::spmm_sparse_dense(csr, B->cols, dview(B), dview(C), accumulate != 0, ctx->stream));
    return MB_OK;
}

int32_t mb_spgemm_dense_out(mb_ctx* ctx, const mb_sparse* A, const mb_sparse* B, mb_block* C, int32_t accumulate) {
    MB_CTX(ctx);
    if (!A || !B || !C) return fail(MB_ERR_INVALID_ARG, "mb_spgemm_dense_out: null argument");
    if (A->cols != B->rows) return fail(MB_ERR_DIM_MISMATCH, "matrix dimension mismatch: %d v.s %d", A->cols, B->rows);
    int32_t r = dense_f64_out(C, A->rows, B->cols, "SparseMatrix.multiply");
    if (r) return r;
    MB_CUDA(mb::spgemm_dense_out(csc(A), csc(B), dview(C), accumulate != 0, ctx->stream));
    return MB_OK;
}

int32_t mb_fill_sparse_uniform(mb_ctx* ctx, mb_sparse* S, int64_t partition_seed) {
    MB_CTX(ctx);
    if (!S) return fail(MB_ERR_INVALID_ARG, "mb_fill_sparse_uniform: null block");
    if (S->cols == 0) {
        if (S->nnz != 0) return fail(MB_ERR_INVALID_ARG, "mb_fill_sparse_uniform: %lld non-zeros in 0 columns", (long long)S->nnz);
        MB_CUDA(cudaMemsetAsync(S->colptr, 0, sizeof(int), ctx->stream));      // colptr = {0}
        return MB_OK;
    }
    if (S->nnz % S->cols != 0)
        return fail(MB_ERR_INVALID_ARG, "mb_fill_sparse_uniform: nnz %lld is not a multiple of cols %d", (long long)S->nnz, S->cols);
    const int s = (int)(S->nnz / S->cols);
    if (s > S->rows) return fail(MB_ERR_INVALID_ARG, "mb_fill_sparse_uniform: %d rows per column of %d", s, S->rows);
    // the row sampling's last stream position must stay within the 2^39 positions the jump tables reach
    if ((long long)S->rows * S->cols + S->nnz >= (1LL << 39))
        return fail(MB_ERR_UNSUPPORTED, "mb_fill_sparse_uniform: a %dx%d block exceeds the generator's 2^39 stream positions",
                    S->rows, S->cols);
    const unsigned long long state0 = (unsigned long long)mb_hash_seed(partition_seed);
    if (S->nnz) {
        MB_CUDA(mb::fill_uniform_f64(S->values, 1, S->nnz, (int)S->nnz, 1, 0, state0, 0, 0.0, 1.0, ctx->stream));
    }
    MB_CUDA(mb::sparse_sample_rows(S->rows, S->cols, s, state0, S->nnz, S->colptr, S->rowidx, ctx->stream));
    return MB_OK;
}

// ------------------------------------------------------------------------------- SparseVecMatrix (matrix/SparseVecMatrix.scala)
// A row shard is the CSC handle of its transpose: colptr = row pointers, rowidx = column ids.
static mb::CsrView rows_of(const mb_sparse* S) { return mb::CsrView{S->cols, S->rows, S->colptr, S->rowidx, S->values}; }

// Gives the handle made by mb_sparse_alloc(nnz = 0) room for nnz entries.
static cudaError_t sparse_reserve(mb_sparse* S, long long nnz) {
    S->nnz = nnz;
    if (!nnz) return cudaSuccess;
    cudaError_t e = cudaMalloc(&S->rowidx, sizeof(int) * (size_t)nnz);
    return e == cudaSuccess ? cudaMalloc(&S->values, sizeof(double) * (size_t)nnz) : e;
}

int32_t mb_spvec_multiply(mb_ctx* ctx, const mb_sparse* A, const mb_sparse* B, mb_sparse** out) {
    if (out) *out = nullptr;
    MB_CTX(ctx);
    if (!A || !B || !out) return fail(MB_ERR_INVALID_ARG, "mb_spvec_multiply: null argument");
    if (A->rows != B->cols)
        return fail(MB_ERR_DIM_MISMATCH, "multiplySparse: this.nCols %d does not match other.nRows %d", A->rows, B->cols);
    mb_sparse* raw = nullptr;
    int32_t r = mb_sparse_alloc(ctx, B->rows, A->cols, 0, &raw);
    if (r) return r;
    SparsePtr R(raw, SparseFree{ctx});
    mb::SpvecWork w;
    long long total = 0;
    cudaError_t e = mb::spvec_count(rows_of(A), rows_of(B), R->colptr, &total, &w, ctx->stream);
    if (e == cudaSuccess && total > 0x7fffffffLL)
        return fail(MB_ERR_UNSUPPORTED, "multiplySparse: the product has %lld entries, more than 2^31 - 1", total);
    if (e == cudaSuccess) e = sparse_reserve(R.get(), total);
    if (e == cudaSuccess && total) e = mb::spvec_fill(rows_of(A), rows_of(B), w, R->colptr, R->rowidx, R->values, ctx->stream);
    if (e != cudaSuccess) return cuda_fail(e, "multiplySparse");
    *out = R.release();
    return MB_OK;
}

int32_t mb_spvec_multiply_host(mb_ctx* ctx, int32_t a_rows, int32_t k, const int32_t* a_rowptr, const int32_t* a_colidx,
                               const double* a_values, int32_t n, const int32_t* b_rowptr, const int32_t* b_colidx,
                               const double* b_values, mb_sparse** out) {
    if (out) *out = nullptr;
    MB_CTX(ctx);
    if (!out || !a_rowptr || !b_rowptr) return fail(MB_ERR_INVALID_ARG, "mb_spvec_multiply_host: null argument");
    mb_sparse *a = nullptr, *b = nullptr, *c = nullptr;
    int32_t r = mb_sparse_upload(ctx, k, a_rows, a_rowptr, a_colidx, a_values, &a);     // the CSC of A's transpose
    if (r == MB_OK) r = mb_sparse_upload(ctx, n, k, b_rowptr, b_colidx, b_values, &b);
    if (r == MB_OK) r = mb_spvec_multiply(ctx, a, b, &c);
    const SparsePtr A(a, SparseFree{ctx}), B(b, SparseFree{ctx});
    SparsePtr C(c, SparseFree{ctx});
    if (r == MB_OK) r = mb_synchronize(ctx);
    if (r == MB_OK) *out = C.release();
    return r;
}

int32_t mb_spvec_coo(mb_ctx* ctx, const mb_sparse* C, int32_t* rows_out, int32_t* cols_out, float* values_out) {
    MB_CTX(ctx);
    if (!C || (C->nnz > 0 && (!rows_out || !cols_out || !values_out))) return fail(MB_ERR_INVALID_ARG, "mb_spvec_coo: null argument");
    std::vector<int32_t> rowptr((size_t)C->cols + 1);
    std::vector<double> vals((size_t)C->nnz);
    int32_t r = mb_sparse_download(ctx, C, rowptr.data(), cols_out, vals.data());
    if (r) return r;
    for (int32_t i = 0; i < C->cols; ++i)
        for (int32_t q = rowptr[i]; q < rowptr[i + 1]; ++q) rows_out[q] = i;
    for (long long q = 0; q < C->nnz; ++q) values_out[q] = (float)vals[q];      // exact: the values are float32 widened
    return MB_OK;
}

int32_t mb_dense_rows_to_sparse(mb_ctx* ctx, const mb_block* rows, mb_sparse** out) {
    if (out) *out = nullptr;
    MB_CTX(ctx);
    if (!rows || !out) return fail(MB_ERR_INVALID_ARG, "mb_dense_rows_to_sparse: null argument");
    if (rows->dtype != MB_F64) return fail(MB_ERR_UNSUPPORTED, "toSparseVecMatrix: fp64 blocks only");
    mb_sparse* raw = nullptr;
    int32_t r = mb_sparse_alloc(ctx, rows->cols, rows->rows, 0, &raw);
    if (r) return r;
    SparsePtr R(raw, SparseFree{ctx});
    long long total = 0;
    cudaError_t e = mb::dense_rows_count(dview(rows), rows->rows, rows->cols, R->colptr, &total, ctx->stream);
    if (e == cudaSuccess && total > 0x7fffffffLL)
        return fail(MB_ERR_UNSUPPORTED, "toSparseVecMatrix: %lld non-zeros, more than 2^31 - 1", total);
    if (e == cudaSuccess) e = sparse_reserve(R.get(), total);
    if (e == cudaSuccess && total)
        e = mb::dense_rows_compact(dview(rows), rows->rows, rows->cols, R->colptr, R->rowidx, R->values, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) return cuda_fail(e, "toSparseVecMatrix");
    *out = R.release();
    return MB_OK;
}

int32_t mb_fill_spvec_uniform(mb_ctx* ctx, mb_sparse* S, int64_t partition_seed, double lo, double hi) {
    MB_CTX(ctx);
    if (!S) return fail(MB_ERR_INVALID_ARG, "mb_fill_spvec_uniform: null block");
    if (S->cols == 0 || S->nnz == 0) {
        if (S->nnz != 0) return fail(MB_ERR_INVALID_ARG, "mb_fill_spvec_uniform: %lld non-zeros in 0 rows", (long long)S->nnz);
        MB_CUDA(cudaMemsetAsync(S->colptr, 0, sizeof(int) * ((size_t)S->cols + 1), ctx->stream));     // s = 0: empty rows
        return MB_OK;
    }
    if (S->nnz % S->cols != 0)
        return fail(MB_ERR_INVALID_ARG, "mb_fill_spvec_uniform: nnz %lld is not a multiple of %d rows", (long long)S->nnz, S->cols);
    const int s = (int)(S->nnz / S->cols);
    if (s > S->rows) return fail(MB_ERR_INVALID_ARG, "mb_fill_spvec_uniform: %d columns per row of %d", s, S->rows);
    if (S->nnz + S->rows >= (1LL << 39))
        return fail(MB_ERR_UNSUPPORTED, "mb_fill_spvec_uniform: %d rows of %d columns exceed the generator's 2^39 stream positions",
                    S->cols, S->rows);
    const unsigned long long state0 = (unsigned long long)mb_hash_seed(partition_seed);
    MB_CUDA(mb::fill_uniform_f64(S->values, 1, S->nnz, (int)S->nnz, 1, 0, state0, 0, lo, hi, ctx->stream));
    // row 0's columns: one "column" of the sampler over nColumns positions, from position s*P
    MB_CUDA(mb::sparse_sample_rows(S->rows, 1, s, state0, S->nnz, S->colptr, S->rowidx, ctx->stream));
    MB_CUDA(mb::spvec_replicate_columns(S->cols, s, S->colptr, S->rowidx, ctx->stream));
    return MB_OK;
}

int32_t mb_fill_spvec_normal(mb_ctx* ctx, mb_sparse* S, int64_t partition_seed, double mean, double variance) {
    MB_CTX(ctx);
    if (!S) return fail(MB_ERR_INVALID_ARG, "mb_fill_spvec_normal: null block");
    if (S->cols == 0 || S->nnz == 0) {
        if (S->nnz != 0) return fail(MB_ERR_INVALID_ARG, "mb_fill_spvec_normal: %lld non-zeros in 0 rows", (long long)S->nnz);
        MB_CUDA(cudaMemsetAsync(S->colptr, 0, sizeof(int) * ((size_t)S->cols + 1), ctx->stream));     // s = 0: empty rows
        return MB_OK;
    }
    if (S->nnz % S->cols != 0)
        return fail(MB_ERR_INVALID_ARG, "mb_fill_spvec_normal: nnz %lld is not a multiple of %d rows", (long long)S->nnz, S->cols);
    const int s = (int)(S->nnz / S->cols);
    if (s > S->rows) return fail(MB_ERR_INVALID_ARG, "mb_fill_spvec_normal: %d columns per row of %d", s, S->rows);
    int64_t positions = 0;
    const int32_t r = fill_normal(ctx, S->values, 1, S->nnz, (int)S->nnz, 1, 0, partition_seed, mean, variance, S->rows,
                                  &positions, "mb_fill_spvec_normal");
    if (r) return r;
    // row 0's columns: one "column" of the sampler over nColumns positions, from the first position the values left
    const unsigned long long state0 = (unsigned long long)mb_hash_seed(partition_seed);
    MB_CUDA(mb::sparse_sample_rows(S->rows, 1, s, state0, positions, S->colptr, S->rowidx, ctx->stream));
    MB_CUDA(mb::spvec_replicate_columns(S->cols, s, S->colptr, S->rowidx, ctx->stream));
    return MB_OK;
}

// ------------------------------------------------------------------------------------------ PageRank (examples/PageRank.scala)
// A vector of the step: an fp64 block of `len` rows and one column, element i at p[i * stride].
static int32_t pagerank_vector(const mb_block* v, int len, const char* what, double** p) {
    if (!v) return fail(MB_ERR_INVALID_ARG, "PageRank: null %s", what);
    if (v->dtype != MB_F64) return fail(MB_ERR_UNSUPPORTED, "PageRank: %s must be fp64", what);
    if (v->cols != 1 || v->rows != len)
        return fail(MB_ERR_DIM_MISMATCH, "PageRank: %s is %dx%d, expected %dx1", what, v->rows, v->cols, len);
    if (len > 1 && rs(v) != 1) return fail(MB_ERR_UNSUPPORTED, "PageRank: %s must be contiguous", what);
    *p = f64_ptr(v);
    return MB_OK;
}

// The in-link rows of a handle, binned on first use (the list stays with the handle: blocks are immutable values).
static int32_t pagerank_links_of(mb_ctx* ctx, mb_sparse* L, int64_t seg_len, mb::PagerankPlan* plan) {
    if (!L) return fail(MB_ERR_INVALID_ARG, "PageRank: null in-links");
    if (seg_len <= 0) return fail(MB_ERR_INVALID_ARG, "PageRank: segment length %lld must be positive", (long long)seg_len);
    if (L->pagerank_nheavy < 0) {
        mb::PagerankPlan p;
        cudaError_t e = mb::pagerank_plan(rows_of(L), L->nnz, &p, ctx->stream);
        if (e != cudaSuccess) {
            cudaFree(p.heavy);
            return cuda_fail(e, "PageRank: binning the in-links");
        }
        L->pagerank_heavy = p.heavy;
        L->pagerank_nheavy = p.nheavy;
    }
    plan->heavy = L->pagerank_heavy;
    plan->nheavy = L->pagerank_nheavy;
    return MB_OK;
}

int32_t mb_pagerank_step(mb_ctx* ctx, mb_sparse* in_links, const mb_block* x, int64_t seg_len, double addend, mb_block* y) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    if (!in_links) return fail(MB_ERR_INVALID_ARG, "PageRank: null in-links");
    double *xp = nullptr, *yp = nullptr;
    int32_t r = pagerank_vector(x, in_links->rows, "x", &xp);
    if (r == MB_OK) r = pagerank_vector(y, in_links->cols, "y", &yp);
    if (r) return r;
    if (in_links->rows && in_links->cols && xp < yp + in_links->cols && yp < xp + in_links->rows)
        return fail(MB_ERR_INVALID_ARG, "PageRank: y overlaps x");
    mb::PagerankPlan plan;
    if ((r = pagerank_links_of(ctx, in_links, seg_len, &plan)) != MB_OK) return r;
    MB_CUDA(mb::pagerank_step(rows_of(in_links), plan, xp, seg_len, addend, yp, ctx->stream));
    return MB_OK;
}

int32_t mb_pagerank_train(mb_ctx* ctx, mb_sparse* in_links, int64_t seg_len, double addend, int32_t iterations,
                          mb_block* x_inout) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    if (!in_links) return fail(MB_ERR_INVALID_ARG, "PageRank: null in-links");
    if (in_links->rows != in_links->cols)
        return fail(MB_ERR_DIM_MISMATCH, "PageRank: %d target rows over %d sources: the loop needs a square link matrix",
                    in_links->cols, in_links->rows);
    double* xp = nullptr;
    int32_t r = pagerank_vector(x_inout, in_links->rows, "x", &xp);
    if (r) return r;
    mb::PagerankPlan plan;
    if ((r = pagerank_links_of(ctx, in_links, seg_len, &plan)) != MB_OK) return r;
    const int n = in_links->rows;
    if (iterations <= 0 || n == 0) return MB_OK;
    mb::StreamBuffer scratch;
    MB_CUDA(scratch.alloc(sizeof(double) * (size_t)n, ctx->stream));
    double *cur = xp, *next = scratch.as<double>();
    cudaError_t e = cudaSuccess;
    for (int it = 0; it < iterations && e == cudaSuccess; ++it) {
        e = mb::pagerank_step(rows_of(in_links), plan, cur, seg_len, addend, next, ctx->stream);
        std::swap(cur, next);
    }
    if (e == cudaSuccess && cur != xp) e = cudaMemcpyAsync(xp, cur, sizeof(double) * (size_t)n, cudaMemcpyDeviceToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    return e == cudaSuccess ? MB_OK : cuda_fail(e, "mb_pagerank_train");
}

int32_t mb_pagerank_host(mb_ctx* ctx, int32_t n, int64_t num_rows, const int64_t* ids, const int64_t* rowptr,
                         const int32_t* targets, const double* values, double damping, int64_t seg_len, double addend,
                         int32_t iterations, double* ranks_inout) {
    MB_CTX(ctx);
    if (n < 0 || num_rows < 0 || !rowptr || (n > 0 && !ranks_inout)) return fail(MB_ERR_INVALID_ARG, "mb_pagerank_host: bad argument");
    if (num_rows > 0 && rowptr[num_rows] < 0) return fail(MB_ERR_INVALID_ARG, "mb_pagerank_host: bad row pointers");
    const size_t cap = num_rows > 0 ? (size_t)std::max<int64_t>(rowptr[num_rows], 0) : 0;
    std::vector<int32_t> in_rowptr((size_t)n + 1), sources(std::max<size_t>(cap, 1));
    std::vector<double> weights(std::max<size_t>(cap, 1));
    int64_t nnz = 0;
    int32_t r = mb_pagerank_links(n, num_rows, ids, rowptr, targets, values, 0, n, damping, in_rowptr.data(), sources.data(),
                                  weights.data(), &nnz);
    if (r || n == 0) return r;
    mb_sparse* l = nullptr;
    mb_block* xb = nullptr;
    if ((r = mb_sparse_upload(ctx, n, n, in_rowptr.data(), sources.data(), weights.data(), &l)) != MB_OK) return r;
    const SparsePtr L(l, SparseFree{ctx});
    if ((r = mb_block_alloc(ctx, n, 1, MB_F64, &xb)) != MB_OK) return r;
    const BlockPtr x(xb, BlockFree{ctx});
    cudaError_t e = cudaMemcpy(f64_ptr(xb), ranks_inout, sizeof(double) * (size_t)n, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) return cuda_fail(e, "mb_pagerank_host");
    if ((r = mb_pagerank_train(ctx, l, seg_len, addend, iterations, xb)) != MB_OK) return r;
    e = cudaMemcpy(ranks_inout, f64_ptr(xb), sizeof(double) * (size_t)n, cudaMemcpyDeviceToHost);
    return e == cudaSuccess ? MB_OK : cuda_fail(e, "mb_pagerank_host");
}

// ------------------------------------------------------------------------------ NeuralNetwork (examples/NeuralNetwork.scala)
int32_t mb_nn_labels_upload(mb_ctx* ctx, const int32_t* labels, int64_t count, void** labels_out) {
    if (labels_out) *labels_out = nullptr;
    MB_CTX(ctx);
    if (!labels || !labels_out || count <= 0) return fail(MB_ERR_INVALID_ARG, "mb_nn_labels_upload: null or empty labels");
    for (int64_t i = 0; i < count; ++i)
        if (labels[i] < 0 || labels[i] >= mb::NN_CLASSES)
            return fail(MB_ERR_INVALID_ARG, "NeuralNetwork: label %d of row %lld is outside 0..%d", labels[i], (long long)i, mb::NN_CLASSES - 1);
    void* d = nullptr;
    MB_CUDA(cudaMalloc(&d, sizeof(int32_t) * (size_t)count));
    const cudaError_t e = cudaMemcpy(d, labels, sizeof(int32_t) * (size_t)count, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        cudaFree(d);
        return cuda_fail(e, "mb_nn_labels_upload");
    }
    *labels_out = d;
    return MB_OK;
}

int32_t mb_nn_labels_free(mb_ctx* ctx, void* labels) {
    MB_CTX(ctx);
    MB_CUDA(cudaFree(labels));
    return MB_OK;
}

// A column-major fp64 block of the given shape, or the error that says what it is instead.
static int32_t nn_colmajor(const mb_block* b, int rows, int cols, const char* what) {
    if (!b) return fail(MB_ERR_INVALID_ARG, "NeuralNetwork: null %s", what);
    if (b->dtype != MB_F64) return fail(MB_ERR_UNSUPPORTED, "NeuralNetwork: %s must be fp64", what);
    if (b->rows != rows || b->cols != cols)
        return fail(MB_ERR_DIM_MISMATCH, "NeuralNetwork: %s is %dx%d, expected %dx%d", what, b->rows, b->cols, rows, cols);
    if (b->is_transpose) return fail(MB_ERR_UNSUPPORTED, "NeuralNetwork: %s must be column-major", what);
    return MB_OK;
}

// Rows [k0, k1) of block b's D1 against columns [k0, k1) of its XT: one entry of the grouped launch, one partial.
struct NnChunk { int b, k0, k1; };

// Steps 1-5 of an iteration for the blocks given.  out1 / out2 non-null: the gradient sums go there; null: W1 and W2 are updated.
static int32_t nn_run(mb_ctx* ctx, const mb_block* const* X, const mb_block* const* XT, const void* const* labels, int nsel,
                      const mb_block* W1, const mb_block* W2, double scale, mb_block* out1, mb_block* out2,
                      mb_block* const* D1_out, bool update) {
    if (!X || !labels || nsel <= 0) return fail(MB_ERR_INVALID_ARG, "NeuralNetwork: no selected blocks");
    if (!W1 || !W2) return fail(MB_ERR_INVALID_ARG, "NeuralNetwork: null weight");
    const int V = W1->rows, H = W1->cols;
    if (V <= 0 || H <= 0) return fail(MB_ERR_INVALID_ARG, "NeuralNetwork: the hidden weight is %dx%d", V, H);
    int32_t r = nn_colmajor(W1, V, H, "the hidden weight");
    if (r == MB_OK) r = nn_colmajor(W2, H, mb::NN_CLASSES, "the output weight");
    if (r == MB_OK && !update) r = nn_colmajor(out1, V, H, "the hidden-weight gradient");
    if (r == MB_OK && !update) r = nn_colmajor(out2, H, mb::NN_CLASSES, "the output-weight gradient");
    if (r) return r;
    for (int b = 0; b < nsel; ++b) {
        if (!X[b] || !labels[b]) return fail(MB_ERR_INVALID_ARG, "NeuralNetwork: block %d or its labels are null", b);
        if (X[b]->dtype != MB_F64) return fail(MB_ERR_UNSUPPORTED, "NeuralNetwork: fp64 blocks only (block %d)", b);
        if (X[b]->rows <= 0) return fail(MB_ERR_INVALID_ARG, "NeuralNetwork: block %d has no rows", b);
        if (X[b]->cols != V)
            return fail(MB_ERR_DIM_MISMATCH, "NeuralNetwork: block %d has %d columns, the hidden weight %d rows", b, X[b]->cols, V);
        if (XT && XT[b]) {
            if (XT[b]->dtype != MB_F64) return fail(MB_ERR_UNSUPPORTED, "NeuralNetwork: fp64 blocks only (transposed block %d)", b);
            if (XT[b]->rows != V || XT[b]->cols != X[b]->rows)
                return fail(MB_ERR_DIM_MISMATCH, "NeuralNetwork: transposed block %d is %dx%d, expected %dx%d", b, XT[b]->rows,
                            XT[b]->cols, V, X[b]->rows);
        }
        if (D1_out && D1_out[b] && (r = nn_colmajor(D1_out[b], X[b]->rows, H, "a hidden-delta block")) != MB_OK) return r;
    }
    const int sms = ctx->num_sms;
    const long long ldp = (V + 1) & ~1;                        // leading dimension of a hidden-weight partial
    // chunks of the inner dimension: enough entries to give every SM a tile, at least 512 rows each, starting at multiples
    // of 16 rows so that a chunk of D1 is as aligned as the block
    const int tiles_per = ((V + 127) / 128) * ((H + 127) / 128);
    const int per_block = std::max(1, ((sms + tiles_per - 1) / tiles_per + nsel - 1) / nsel);
    std::vector<NnChunk> chunks;
    std::vector<int> first1(1, 0), first2(1, 0);
    std::vector<size_t> z_off(nsel), p2_off(nsel);
    std::vector<char> grouped(nsel);
    size_t doubles = 0;
    for (int b = 0; b < nsel; ++b) {
        const int rb = X[b]->rows;
        z_off[b] = doubles;
        doubles += (size_t)((rb + 1) & ~1) * H;
    }
    for (int b = 0; b < nsel; ++b) {
        p2_off[b] = doubles;
        const int parts = mb::nn_parts(X[b]->rows, sms);
        doubles += (size_t)parts * H * mb::NN_CLASSES;
        first2.push_back(first2.back() + parts);
    }
    for (int b = 0; b < nsel; ++b) {
        const int rb = X[b]->rows;
        const mb_block* d1 = D1_out ? D1_out[b] : nullptr;
        grouped[b] = XT && XT[b] && !XT[b]->is_transpose && mb::gemm_f64_tma_eligible(f64_ptr(XT[b]), XT[b]->ld, f64_ptr(XT[b]), 2) &&
                     (!d1 || mb::gemm_f64_tma_eligible(f64_ptr(d1), d1->ld, f64_ptr(d1), 2));
        const int n = grouped[b] ? std::max(1, std::min(per_block, rb / 512)) : 1;
        const int len = (((rb + n - 1) / n) + 15) & ~15;
        for (int k0 = 0; k0 < rb; k0 += len) chunks.push_back(NnChunk{b, k0, std::min(rb, k0 + len)});
        first1.push_back((int)chunks.size());
    }
    const size_t p1_off = doubles;
    doubles += chunks.size() * (size_t)ldp * H;
    mb::StreamBuffer ws, idx;
    MB_CUDA(ws.alloc(doubles * sizeof(double), ctx->stream));
    std::vector<int> firsts(first1);
    firsts.insert(firsts.end(), first2.begin(), first2.end());
    MB_CUDA(idx.upload(firsts.data(), firsts.size() * sizeof(int), ctx->stream));
    double* base = ws.as<double>();
    cudaError_t e = cudaSuccess;
    // Z1_b = X_b W1, then the fused output layer and both deltas; D1_b replaces Z1_b unless the caller wants it elsewhere
    for (int b = 0; b < nsel && e == cudaSuccess; ++b) {
        const int rb = X[b]->rows;
        const long long ldz = (rb + 1) & ~1;
        double* z = base + z_off[b];
        e = mb::gemm_f64(X[b]->is_transpose, false, rb, H, V, 1.0, f64_ptr(X[b]), X[b]->ld, f64_ptr(W1), W1->ld, 0.0, z, ldz, sms,
                         ctx->stream, false);
        if (e != cudaSuccess) break;
        const mb_block* d1 = D1_out ? D1_out[b] : nullptr;
        e = mb::nn_backprop_f64(z, ldz, rb, H, f64_ptr(W2), W2->ld, static_cast<const int*>(labels[b]), d1 ? f64_ptr(d1) : z,
                                d1 ? d1->ld : ldz, base + p2_off[b], sms, ctx->stream);
    }
    // X_b^T D1_b: the chunks of the blocks with a usable XT as entries of grouped launches, the other blocks one GEMM each
    static thread_local mb::G2Launch L;
    L = mb::G2Launch();
    for (size_t c = 0; c < chunks.size() && e == cudaSuccess; ++c) {
        const NnChunk& ch = chunks[c];
        const mb_block* d1b = D1_out ? D1_out[ch.b] : nullptr;
        const double* d1 = d1b ? f64_ptr(d1b) : base + z_off[ch.b];
        const long long ldd = d1b ? d1b->ld : (X[ch.b]->rows + 1) & ~1;
        double* P = base + p1_off + c * (size_t)ldp * H;
        if (!grouped[ch.b]) {
            const mb_block* x = X[ch.b];
            e = mb::gemm_f64(!x->is_transpose, false, V, H, x->rows, 1.0, f64_ptr(x), x->ld, d1, ldd, 0.0, P, ldp, sms, ctx->stream,
                             false);
            continue;
        }
        mb::G2Operand& A = L.A[L.na];
        A.ptr = f64_ptr(XT[ch.b]) + (long long)ch.k0 * XT[ch.b]->ld; A.ld = XT[ch.b]->ld; A.rows = V; A.cols = ch.k1 - ch.k0;
        mb::G2Operand& B = L.B[L.nb];
        B.ptr = d1 + ch.k0; B.ld = ldd; B.rows = ch.k1 - ch.k0; B.cols = H;
        mb::G2Entry& en = L.E[L.ne++];
        en.nseg = 1; en.a_op[0] = L.na++; en.b_op[0] = L.nb++;
        en.M = V; en.N = H; en.D = P; en.ldd = ldp;
        if (L.ne == mb::G2_MAX_OPS) {
            e = mb::gemm_f64_grouped2(L, sms, ctx->stream);
            L = mb::G2Launch();
        }
    }
    if (e == cudaSuccess && L.ne > 0) e = mb::gemm_f64_grouped2(L, sms, ctx->stream);
    const int* first = idx.as<int>();
    if (e == cudaSuccess)
        e = mb::nn_apply_f64(base + p1_off, ldp, ldp * H, first, nsel, V, H, scale, update ? nullptr : f64_ptr(out1),
                             update ? 0 : out1->ld, update ? f64_ptr(W1) : nullptr, W1->ld, ctx->stream);
    if (e == cudaSuccess)
        e = mb::nn_apply_f64(base + p2_off[0], H, (long long)H * mb::NN_CLASSES, first + nsel + 1, nsel, H, mb::NN_CLASSES, scale,
                             update ? nullptr : f64_ptr(out2), update ? 0 : out2->ld, update ? f64_ptr(W2) : nullptr, W2->ld,
                             ctx->stream);
    return e == cudaSuccess ? MB_OK : cuda_fail(e, "NeuralNetwork");
}

int32_t mb_nn_gradient(mb_ctx* ctx, const mb_block* const* X, const mb_block* const* XT, const void* const* labels,
                       int32_t nsel, const mb_block* W1, const mb_block* W2, double scale, mb_block* dW1_out,
                       mb_block* dW2_out, mb_block* const* D1_out) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    return nn_run(ctx, X, XT, labels, nsel, W1, W2, scale, dW1_out, dW2_out, D1_out, false);
}

int32_t mb_nn_step(mb_ctx* ctx, const mb_block* const* X, const mb_block* const* XT, const void* const* labels, int32_t nsel,
                   mb_block* W1, mb_block* W2, double scale) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    return nn_run(ctx, X, XT, labels, nsel, W1, W2, scale, nullptr, nullptr, nullptr, true);
}

// ------------------------------------------------------------------------------------------- matrix text files (SURVEY 8 f3)
// One part file: the segments' text through mb::save_text.  The file is opened (truncated) before anything else, so an
// unwritable path fails without touching the device.
static int32_t save_segments(mb_ctx* ctx, const mb::TextSegment* segs, const long long* const* host_ids, int count,
                             const char* path, const char* what) {
    FILE* f = std::fopen(path, "wb");
    if (!f) return fail(MB_ERR_IO, "%s: cannot open %s: %s", what, path, std::strerror(errno));
    mb::TextIo io{ctx->stream, nullptr, {}, f};
    cudaError_t e = ensure_copy_streams(ctx);
    for (int i = 0; i < 4 && e == cudaSuccess; ++i) e = next_event(ctx, &io.events[i]);
    int io_errno = 0;
    if (e == cudaSuccess) {
        io.copy_stream = ctx->d2h_stream;
        e = mb::save_text(segs, host_ids, count, io, &io_errno);
    }
    const bool closed = std::fclose(f) == 0;
    if (e != cudaSuccess) return cuda_fail(e, what);
    if (io_errno || !closed) return fail(MB_ERR_IO, "%s: cannot write %s: %s", what, path, std::strerror(io_errno ? io_errno : errno));
    return MB_OK;
}

static mb::TextSegment text_segment(const mb_block* b) {
    return mb::TextSegment{elem_ptr(b), rs(b), cs(b), b->rows, b->cols, b->dtype, nullptr, 0, 0};
}

// DenseVecMatrix.scala:1042-1046: rdd.map(t => t._1 + ":" + t._2.toString).saveAsTextFile(path), one partition
int32_t mb_save_rows(mb_ctx* ctx, const mb_block* rows, const int64_t* row_ids, const char* path) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    if (!path || (rows && rows->rows > 0 && !row_ids) || (rows && (rows->rows < 0 || rows->cols < 0)))
        return fail(MB_ERR_INVALID_ARG, "mb_save_rows: bad argument");
    ctx->events_used = 0;
    mb::TextSegment seg{};
    const long long* host_ids = reinterpret_cast<const long long*>(row_ids);
    mb::StreamBuffer ids;
    const int count = rows && rows->rows > 0 ? 1 : 0;
    if (count) {
        seg = text_segment(rows);
        MB_CUDA(ids.upload(row_ids, sizeof(long long) * (size_t)rows->rows, ctx->stream));
        seg.ids = ids.as<long long>();
    }
    return save_segments(ctx, &seg, &host_ids, count, path, "mb_save_rows");
}

// BlockMatrix.scala:550-555: blocks.map(t => t._1.row + "-" + t._1.column + "-" + t._2.rows + "-" + t._2.cols + ":" +
// t._2.data.mkString(",")).saveAsTextFile(path), one partition (data: the column-major array)
int32_t mb_save_blocks(mb_ctx* ctx, const mb_block* const* blocks, const int32_t* block_rc, int32_t count, const char* path) {
    MB_CTX(ctx);
    MB_LOCK(ctx);
    if (!path || count < 0 || (count > 0 && (!blocks || !block_rc))) return fail(MB_ERR_INVALID_ARG, "mb_save_blocks: bad argument");
    std::vector<mb::TextSegment> segs;
    for (int i = 0; i < count; ++i) {
        if (!blocks[i]) return fail(MB_ERR_INVALID_ARG, "mb_save_blocks: block %d is null", i);
        segs.push_back(text_segment(blocks[i]));
        segs.back().block_row = block_rc[2 * i];
        segs.back().block_col = block_rc[2 * i + 1];
    }
    ctx->events_used = 0;
    std::vector<const long long*> host_ids((size_t)count, nullptr);
    return save_segments(ctx, segs.data(), host_ids.data(), count, path, "mb_save_blocks");
}

}  // extern "C"

// Internal definitions shared by the translation units behind the C ABI (capi.cu, dist.cu): the context and block
// records, error plumbing and small helpers.  Not installed; include/marlin_b200.h is the public surface.
#pragma once
#include "../../include/marlin_b200.h"
#include "gemm_f64.h"
#include "launch.h"
#include "stream_buffer.h"

#include <cuda_runtime.h>
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <mutex>
#include <vector>

struct mb_ctx {
    int device = 0;
    int num_sms = 132;
    cudaStream_t own_stream = nullptr;
    cudaStream_t stream = nullptr;
    std::atomic<long long> launches{0};
    double* scratch = nullptr;          // sum partials + result
    double* host_scalar = nullptr;      // pinned
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    // pipelined host<->device path (mb_matmul_blocked_host): copy streams + a grow-only device workspace
    cudaStream_t h2d_stream = nullptr, d2h_stream = nullptr;
    void* workspace = nullptr;
    size_t workspace_bytes = 0;
    // fp64 mode (mb_set_fp64_mode) and the digit-plane workspace of the int8-split path
    int fp64_mode = MB_FP64_NATIVE;
    int fp64_slices = 7;
    int fp64_bits = 7;
    bool dmma_reference = false;        // mb_set_dmma_reference: the m8n8k4 instances of the fp64 DMMA kernels
    void* ozaki_ws = nullptr;
    size_t ozaki_ws_bytes = 0;
    // partial vectors of the matrix x vector kernels (grow-only)
    double* vec_ws = nullptr;
    size_t vec_ws_bytes = 0;
    // pivots / permutation / info of the factorization entries (grow-only) + a pinned mirror for the results
    int* int_ws = nullptr;
    size_t int_ws_bytes = 0;
    int* int_host = nullptr;
    size_t int_host_count = 0;
    // Events of the host pipelines and the multi-GPU entries (next_event).  An entry resets events_used when it starts,
    // under the lock; re-recording an event is safe because a stream wait binds to the record current when it is issued.
    std::vector<cudaEvent_t> events;
    size_t events_used = 0;
    // Entry points that use the context's own scratch buffers, workspaces, events or copy streams take this lock, so
    // threads sharing one context (Spark local[N] task threads) serialise there; kernel-only entries (gemm, element-wise,
    // transpose, fill) touch no shared host state and need none.  Threads that want concurrency use one context each.
    std::recursive_mutex mu;
};

struct mb_block {
    void* data = nullptr;      // device base pointer (element 0 of the underlying array)
    long long offset = 0;      // in elements
    int rows = 0, cols = 0;    // logical dims
    int ld = 0;                // majorStride
    int is_transpose = 0;
    int dtype = MB_F64;
    int owns = 0;
    int device = 0;
    void* ready_event = nullptr;   // optional cudaEvent_t: the block's contents are final once it has completed
};

// A CSC block (column j: rowidx/values[colptr[j] .. colptr[j+1]), rows strictly increasing).  The CSR copy that the
// sparse x dense product reads is built on first use and kept with the handle: blocks are immutable values.
struct mb_sparse {
    int rows = 0, cols = 0;
    long long nnz = 0;
    int* colptr = nullptr;
    int* rowidx = nullptr;
    double* values = nullptr;
    int owns = 0;
    int device = 0;
    int* csr_rowptr = nullptr;      // owned by the handle
    int* csr_colidx = nullptr;
    double* csr_values = nullptr;
    int* pagerank_heavy = nullptr;  // owned by the handle: the rows mb_pagerank_step gives a warp each (mb::pagerank_plan)
    int pagerank_nheavy = -1;       // -1: not binned yet
};

namespace mb {
cudaError_t ipc_export(const void* dptr, unsigned char handle[64], long long* offset, long long* alloc_bytes);
cudaError_t ipc_open(const unsigned char handle[64], void** base_out);
cudaError_t ipc_open_ex(const unsigned char handle[64], void** base_out, bool pinned);
unsigned long long ipc_evictions();
cudaError_t ipc_close(const unsigned char handle[64]);
cudaError_t ipc_close_all();
cudaError_t flag_signal(void* flag, unsigned long long v, cudaStream_t st);
bool stream_memops_available();
cudaError_t stream_write64(void* flag, unsigned long long v, cudaStream_t st);
cudaError_t stream_wait64_geq(const void* flag, unsigned long long v, cudaStream_t st);
cudaError_t flag_wait(const void* flag, unsigned long long v, cudaStream_t st);
}  // namespace mb

// thread-local message of the last failing call (defined in capi.cu)
int32_t mb_fail(int32_t code, const char* fmt, ...);
#define fail mb_fail
inline int32_t cuda_fail(cudaError_t e, const char* what) {
    return fail(e == cudaErrorMemoryAllocation ? MB_ERR_OOM : MB_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
}
#define MB_CUDA(call)                                       \
    do {                                                    \
        cudaError_t _e = (call);                            \
        if (_e != cudaSuccess) return cuda_fail(_e, #call); \
    } while (0)

inline size_t elem_size(int dtype) { return dtype == MB_F64 ? 8 : (dtype == MB_F32 ? 4 : 2); }
inline char* elem_ptr(const mb_block* b) { return static_cast<char*>(b->data) + b->offset * (long long)elem_size(b->dtype); }
inline double* f64_ptr(const mb_block* b) { return reinterpret_cast<double*>(elem_ptr(b)); }
// strides of the logical (rows x cols) view
inline long long rs(const mb_block* b) { return b->is_transpose ? b->ld : 1; }
inline long long cs(const mb_block* b) { return b->is_transpose ? 1 : b->ld; }
// A block record over device memory the call holds: it owns nothing and lives on the caller's frame.
inline mb_block block_view(void* data, int rows, int cols, int ld, bool row_major, int dtype, int device) {
    mb_block b;
    b.data = data; b.rows = rows; b.cols = cols; b.ld = ld; b.is_transpose = row_major; b.dtype = dtype; b.device = device;
    return b;
}

inline int32_t check_ctx(mb_ctx* ctx) {
    if (!ctx) return fail(MB_ERR_INVALID_ARG, "null context");
    cudaError_t e = cudaSetDevice(ctx->device);
    if (e != cudaSuccess) return cuda_fail(e, "cudaSetDevice");
    mb::begin_call(&ctx->launches, ctx->dmma_reference);    // the launches of this call are counted on, and follow, ctx
    return MB_OK;
}
#define MB_CTX(ctx)                        \
    do {                                   \
        int32_t _r = check_ctx(ctx);       \
        if (_r != MB_OK) return _r;        \
    } while (0)
#define MB_LOCK(ctx) std::lock_guard<std::recursive_mutex> _mb_lock((ctx)->mu)

// The copy streams of the host pipelines, created on first use.
inline cudaError_t ensure_copy_streams(mb_ctx* ctx) {
    if (ctx->h2d_stream) return cudaSuccess;
    cudaError_t e = cudaStreamCreateWithFlags(&ctx->h2d_stream, cudaStreamNonBlocking);
    return e == cudaSuccess ? cudaStreamCreateWithFlags(&ctx->d2h_stream, cudaStreamNonBlocking) : e;
}

// The next unused event of the context's pool, created when the pool runs out.
inline cudaError_t next_event(mb_ctx* ctx, cudaEvent_t* ev) {
    if (ctx->events_used == ctx->events.size()) {
        cudaEvent_t fresh = nullptr;
        cudaError_t e = cudaEventCreateWithFlags(&fresh, cudaEventDisableTiming);
        if (e != cudaSuccess) return e;
        ctx->events.push_back(fresh);
    }
    *ev = ctx->events[ctx->events_used++];
    return cudaSuccess;
}

// A grow-only device buffer: when `need` exceeds *have bytes, the old buffer is freed once the work that may still use
// it has finished (*sync, or the whole device when sync is null) and a buffer of `need` bytes takes its place.
template <class T>
cudaError_t grow(T** p, size_t* have, size_t need, const cudaStream_t* sync) {
    if (need <= *have) return cudaSuccess;
    if (*p) {
        cudaError_t e = sync ? cudaStreamSynchronize(*sync) : cudaDeviceSynchronize();
        if (e != cudaSuccess) return e;
        cudaFree(*p);
        *p = nullptr;
        *have = 0;
    }
    cudaError_t e = cudaMalloc(p, need);
    if (e == cudaSuccess) *have = need;
    return e;
}


// Peer-memory plumbing for the multi-GPU multiply (one process per GPU on one NVSwitch box):
// CUDA IPC mapping of another rank's device buffers, stream-ordered flags in (peer) device memory, and DMA
// copies.  With these the tile replication of BlockMatrix.multiply (matrix/BlockMatrix.scala:161-171) becomes
// copy-engine pulls over NVLink that overlap the first GEMM chunks, and the partial products of the reduceByKey
// (:177) are written by the GEMM epilogue straight into the reducing rank's HBM (P2P stores), with no NCCL call
// on the data path.
#include "../../include/marlin_b200.h"
#include "launch.h"
#include <cuda.h>
#include <cuda_runtime.h>
#include <atomic>
#include <cstring>
#include <map>
#include <mutex>
#include <string>

namespace mb {

namespace {

__global__ void flag_signal_kernel(unsigned long long* flag, unsigned long long v) {
    __threadfence_system();
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(flag), "l"(v) : "memory");
}
__global__ void flag_wait_kernel(const unsigned long long* flag, unsigned long long v) {
    for (;;) {
        unsigned long long cur;
        asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(cur) : "l"(flag) : "memory");
        if (cur >= v) return;
        __nanosleep(256);
    }
}

std::mutex g_mu;
struct Mapping { void* base; bool pinned; unsigned long long last_use; };
std::map<std::string, Mapping> g_opened;   // IPC handle bytes -> mapped base address (per process)
unsigned long long g_use_clock = 0;
std::atomic<unsigned long long> g_evictions{0};

typedef CUresult (*GetRangeFn)(CUdeviceptr*, size_t*, CUdeviceptr);
GetRangeFn get_range_fn() {
    static GetRangeFn fn = nullptr;
    if (!fn) {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuMemGetAddressRange", &ptr, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<GetRangeFn>(ptr);
    }
    return fn;
}

}  // namespace

cudaError_t ipc_export(const void* dptr, unsigned char handle[64], long long* offset, long long* alloc_bytes) {
    GetRangeFn fn = get_range_fn();
    if (!fn) return cudaErrorNotSupported;
    CUdeviceptr base = 0;
    size_t size = 0;
    if (fn(&base, &size, reinterpret_cast<CUdeviceptr>(dptr)) != CUDA_SUCCESS) return cudaErrorInvalidValue;
    cudaIpcMemHandle_t h;
    cudaError_t e = cudaIpcGetMemHandle(&h, reinterpret_cast<void*>(base));
    if (e != cudaSuccess) return e;
    static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
    std::memcpy(handle, &h, 64);
    *offset = static_cast<long long>(reinterpret_cast<CUdeviceptr>(dptr) - base);
    *alloc_bytes = static_cast<long long>(size);
    return cudaSuccess;
}

// Map a peer allocation (cached per handle).  `pinned` mappings (flag arrays, staging buffers) live until ipc_close /
// ipc_close_all; tile mappings are evictable: an exporter that frees a tile and allocates a new one may get the same
// physical allocation back under a NEW handle, which cudaIpcOpenMemHandle refuses while the stale mapping exists
// (cudaErrorAlreadyMapped) — then every evictable mapping is dropped (after a device sync: nothing is in flight on
// them) and the open is retried.  Tile mappings unused for a long time are trimmed as well.
cudaError_t ipc_open_ex(const unsigned char handle[64], void** base_out, bool pinned) {
    std::lock_guard<std::mutex> lk(g_mu);
    std::string key(reinterpret_cast<const char*>(handle), 64);
    ++g_use_clock;
    auto it = g_opened.find(key);
    if (it != g_opened.end()) {
        it->second.last_use = g_use_clock;
        it->second.pinned = it->second.pinned || pinned;
        *base_out = it->second.base;
        return cudaSuccess;
    }
    cudaIpcMemHandle_t h;
    std::memcpy(&h, handle, 64);
    void* base = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess);
    if (e == cudaErrorAlreadyMapped) {
        cudaGetLastError();
        cudaDeviceSynchronize();
        ++g_evictions;
        for (auto jt = g_opened.begin(); jt != g_opened.end();) {
            if (!jt->second.pinned) { cudaIpcCloseMemHandle(jt->second.base); jt = g_opened.erase(jt); }
            else ++jt;
        }
        e = cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess);
    }
    if (e != cudaSuccess) return e;
    g_opened[key] = Mapping{base, pinned, g_use_clock};
    *base_out = base;
    if (g_opened.size() > 256) {                     // trim tile mappings that have not been used for a while
        bool synced = false;
        for (auto jt = g_opened.begin(); jt != g_opened.end();) {
            if (!jt->second.pinned && jt->second.last_use + 4096 < g_use_clock) {
                if (!synced) { cudaDeviceSynchronize(); synced = true; ++g_evictions; }
                cudaIpcCloseMemHandle(jt->second.base);
                jt = g_opened.erase(jt);
            } else ++jt;
        }
    }
    return cudaSuccess;
}
cudaError_t ipc_open(const unsigned char handle[64], void** base_out) { return ipc_open_ex(handle, base_out, false); }
// Bumped whenever evictable mappings were dropped: pointers obtained from ipc_open before that are stale.
unsigned long long ipc_evictions() { return g_evictions.load(); }

// Unmap one peer allocation (the exporter is about to free it, e.g. a staging buffer being regrown).
cudaError_t ipc_close(const unsigned char handle[64]) {
    std::lock_guard<std::mutex> lk(g_mu);
    std::string key(reinterpret_cast<const char*>(handle), 64);
    auto it = g_opened.find(key);
    if (it == g_opened.end()) return cudaSuccess;
    cudaError_t e = cudaIpcCloseMemHandle(it->second.base);
    g_opened.erase(it);
    return e;
}

cudaError_t ipc_close_all() {
    std::lock_guard<std::mutex> lk(g_mu);
    for (auto& kv : g_opened) cudaIpcCloseMemHandle(kv.second.base);
    g_opened.clear();
    return cudaSuccess;
}

// ---- stream memory operations: flag writes and waits executed by the front end / copy engines, NOT by kernels ----
// A tiny kernel launched on a side stream while a persistent kernel holds every SM may never be scheduled (measured:
// scripts/probe_copy_under_persistent.cu — a 1-thread kernel submitted right after the resident grid stays blocked until
// that grid retires, and blocks later launches behind it), so nothing the resident GEMM waits for may depend on one.
typedef CUresult (*StreamWrite64Fn)(CUstream, CUdeviceptr, cuuint64_t, unsigned int);
typedef CUresult (*StreamWait64Fn)(CUstream, CUdeviceptr, cuuint64_t, unsigned int);
static StreamWrite64Fn g_write64 = nullptr;
static StreamWait64Fn g_wait64 = nullptr;
bool stream_memops_available() {
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuStreamWriteValue64", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            g_write64 = reinterpret_cast<StreamWrite64Fn>(p);
        p = nullptr;
        if (cudaGetDriverEntryPoint("cuStreamWaitValue64", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            g_wait64 = reinterpret_cast<StreamWait64Fn>(p);
    });
    return g_write64 != nullptr && g_wait64 != nullptr;
}
cudaError_t stream_write64(void* flag, unsigned long long v, cudaStream_t st) {
    if (!stream_memops_available()) return cudaErrorNotSupported;
    return g_write64(st, reinterpret_cast<CUdeviceptr>(flag), v, CU_STREAM_WRITE_VALUE_DEFAULT) == CUDA_SUCCESS ? cudaSuccess : cudaErrorNotSupported;
}
cudaError_t stream_wait64_geq(const void* flag, unsigned long long v, cudaStream_t st) {
    if (!stream_memops_available()) return cudaErrorNotSupported;
    return g_wait64(st, reinterpret_cast<CUdeviceptr>(flag), v, CU_STREAM_WAIT_VALUE_GEQ) == CUDA_SUCCESS ? cudaSuccess : cudaErrorNotSupported;
}

cudaError_t flag_signal(void* flag, unsigned long long v, cudaStream_t st) {
    flag_signal_kernel<<<1, 1, 0, st>>>(static_cast<unsigned long long*>(flag), v);
    return launched();
}
cudaError_t flag_wait(const void* flag, unsigned long long v, cudaStream_t st) {
    flag_wait_kernel<<<1, 1, 0, st>>>(static_cast<const unsigned long long*>(flag), v);
    return launched();
}

}  // namespace mb

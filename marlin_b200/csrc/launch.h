// Kernel launches of the library, counted where they are made.  Every C-ABI entry starts a call on its context
// (check_ctx in internal.h); each kernel the call then enqueues adds one to that context's count (mb_launch_count).
#pragma once
#include <atomic>
#include <cuda_runtime.h>

namespace mb {

// What the C-ABI call running on this thread asks of the launches it makes.
struct Call {
    std::atomic<long long>* count = nullptr;      // the launch count of the call's context
    bool dmma_reference = false;                  // mb_set_dmma_reference: the m8n8k4 instances of the fp64 DMMA kernels
};
inline thread_local Call g_call;

// Set by every C-ABI entry.  Entries nest, but a nested entry always passes its caller's context, so setting it again
// there changes nothing.
inline void begin_call(std::atomic<long long>* count, bool dmma_reference) { g_call = Call{count, dmma_reference}; }

// n kernels enqueued by the current call at once: the kernel nodes of a graph launch.
inline void count_launches(long long n) {
    if (g_call.count) g_call.count->fetch_add(n, std::memory_order_relaxed);
}

// Follows every kernel<<<...>>>: the launch's error, counting the kernel when it was enqueued.
inline cudaError_t launched() {
    const cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) count_launches(1);
    return e;
}

// Kernel<<<grid, threads, smem, stream>>>(args...), raising the kernel's dynamic shared-memory limit to smem on its first
// launch.  Setting the attribute is idempotent, so threads that race on a first launch may both set it.
template <auto Kernel, class... Args>
cudaError_t launch_with_smem(int grid, int threads, int smem, cudaStream_t stream, const Args&... args) {
    static std::atomic<bool> attr_done{false};
    if (!attr_done.load(std::memory_order_acquire)) {
        const cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) return e;
        attr_done.store(true, std::memory_order_release);
    }
    Kernel<<<grid, threads, smem, stream>>>(args...);
    return launched();
}

}  // namespace mb

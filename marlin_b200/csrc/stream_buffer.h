// Device memory for the length of one call: the one owner of every temporary of the C ABI and its kernel launchers, so
// cudaMallocAsync / cudaFreeAsync appear only here.  Memory that outlives the call (handles, context workspaces) stays on
// plain cudaMalloc.
#pragma once
#include <cuda_runtime.h>

namespace mb {

// Taken from the device's default pool in the order of stream `st` and returned in that order when the owner is
// destroyed, so work enqueued on `st` before then still reads valid memory.  Move-only.
class StreamBuffer {
  public:
    StreamBuffer() = default;
    StreamBuffer(StreamBuffer&& o) noexcept : p_(o.p_), st_(o.st_) { o.p_ = nullptr; }
    ~StreamBuffer() { release(); }

    // `bytes` of device memory on `st`; what the owner held before is returned first.
    cudaError_t alloc(size_t bytes, cudaStream_t st) {
        release();
        st_ = st;
        const cudaError_t e = cudaMallocAsync(&p_, bytes, st);
        if (e != cudaSuccess) p_ = nullptr;
        return e;
    }
    // A device copy of `bytes` of host memory, enqueued on `st`.  An empty array still gets 8 bytes, so it has an address.
    cudaError_t upload(const void* host, size_t bytes, cudaStream_t st) {
        const cudaError_t e = alloc(bytes ? bytes : 8, st);
        return e == cudaSuccess && bytes ? cudaMemcpyAsync(p_, host, bytes, cudaMemcpyHostToDevice, st) : e;
    }
    template <class T>
    T* as() const { return static_cast<T*>(p_); }

  private:
    void release() {
        if (p_) cudaFreeAsync(p_, st_);
        p_ = nullptr;
    }
    void* p_ = nullptr;
    cudaStream_t st_ = nullptr;
};

}  // namespace mb

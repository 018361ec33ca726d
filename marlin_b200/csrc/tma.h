// Host side of the TMA GEMMs (gemm_f64.cu, gemm_bf16.cu, gemm_ozaki.cu): tensor maps from the driver's
// cuTensorMapEncodeTiled.
#pragma once
#include <cstdint>
#include <cuda.h>
#include <cuda_runtime.h>

namespace mb {

typedef CUresult (*TmaEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// The driver's cuTensorMapEncodeTiled, looked up once; nullptr when the driver does not provide it.
inline TmaEncodeFn tma_encode_fn() {
    static const TmaEncodeFn fn = [] {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            return reinterpret_cast<TmaEncodeFn>(ptr);
        return TmaEncodeFn(nullptr);
    }();
    return fn;
}

// Tiled tensor map with 128-byte swizzle over a `rank`-dimensional array (2 or 3): dims[0] is the contiguous
// dimension, strides[i] the byte stride of dims[i + 1], and one TMA load moves a box[0] x box[1] (x 1) box.
// Out-of-range elements load as zeros.  False when the driver has no encoder or rejects the map.
inline bool tma_encode(CUtensorMap* map, CUtensorMapDataType type, cuuint32_t rank, const void* base, const cuuint64_t* dims,
                       const cuuint64_t* strides, const cuuint32_t* box) {
    const TmaEncodeFn fn = tma_encode_fn();
    if (!fn) return false;
    const cuuint32_t estr[3] = {1, 1, 1};
    return fn(map, type, rank, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
              CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// 2-D: a d0 x d1 array (d0 contiguous, d1 at byte stride stride1), loaded in box0 x box1 boxes.
inline bool tma_map(CUtensorMap* map, CUtensorMapDataType type, const void* base, uint64_t d0, uint64_t d1, uint64_t stride1,
                    uint32_t box0, uint32_t box1) {
    const cuuint64_t dims[2] = {d0, d1}, strides[1] = {stride1};
    const cuuint32_t box[2] = {box0, box1};
    return tma_encode(map, type, 2, base, dims, strides, box);
}

// 3-D: a d0 x d1 x d2 array (byte strides stride1, stride2), loaded in box0 x box1 x 1 boxes.
inline bool tma_map_3d(CUtensorMap* map, CUtensorMapDataType type, const void* base, uint64_t d0, uint64_t d1, uint64_t d2,
                       uint64_t stride1, uint64_t stride2, uint32_t box0, uint32_t box1) {
    const cuuint64_t dims[3] = {d0, d1, d2}, strides[2] = {stride1, stride2};
    const cuuint32_t box[3] = {box0, box1, 1};
    return tma_encode(map, type, 3, base, dims, strides, box);
}

}  // namespace mb

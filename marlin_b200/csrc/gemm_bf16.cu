// bf16 block GEMM on the Hopper tensor cores (wgmma) — the bf16 flavour of SubMatrix.multiply
// (reference: matrix/SubMatrix.scala:87-91) for BASELINE config 5 (65536^2 bf16, 4x4 grid).
//
//   C (M x N, column-major, fp32 or bf16) = op(A) * op(B) [+ C],  A/B bf16, fp32 accumulation in registers.
//
// Structure (one persistent CTA per SM, 384 threads, 128 x 256 C tile):
//   warpgroup 0     TMA producer : one thread issues cp.async.bulk.tensor.2d tiles (SWIZZLE_128B) into a 4-stage smem ring
//   warpgroups 1,2  consumers    : each issues wgmma.mma_async m64n256k16 (f32 += bf16 x bf16) for its 64 rows of the
//                                  tile, holds the 64 x 256 fp32 accumulator in registers (128 per thread) and stores it
//                                  to global memory after the last k-slab.  One slab's wgmma group stays in flight while
//                                  the next is issued; a stage is handed back once the group that read it has retired.
// setmaxnreg moves registers from the producer warpgroup to the consumers.
//
// Column-major operands map onto wgmma majors without any data movement:
//   A 'N' (M x K, m contiguous)  -> MN-major A : smem atoms [64 k-rows][64 m] (TMA box 64x64), LBO = 8 KiB, SBO = 1 KiB
//   A 'T' (K x M, k contiguous)  -> K-major  A : smem [128 m-rows][64 k]      (TMA box 64x128),            SBO = 1 KiB
//   B 'N' (K x N, k contiguous)  -> K-major  B : smem [256 n-rows][64 k]      (TMA box 64x256)
//   B 'T' (N x K, n contiguous)  -> MN-major B : 4 atoms [64 k-rows][64 n]
#include "gemm_bf16.h"
#include "ptx.cuh"
#include "launch.h"
#include "tma.h"
#include <cuda_bf16.h>

namespace mb {

namespace {

constexpr int BM = 128, BN = 256, BK = 64;
constexpr int A_BYTES = BM * BK * 2;             // 16 KiB
constexpr int B_BYTES = BN * BK * 2;             // 32 KiB
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;   // 48 KiB
constexpr int NUM_STAGES = 4;                    // 192 KiB
constexpr int NUM_CONSUMER_WARPS = 8;
constexpr int NUM_THREADS = 128 + NUM_CONSUMER_WARPS * 32;
constexpr int SMEM_BYTES = NUM_STAGES * STAGE_BYTES + 1024 + 256;
constexpr int BAND = 16;

constexpr int MAX_SEG = 8;
// K segments: C = sum over seg of op(A_seg) * op(B_seg).  One segment for a plain GEMM; k of them when the kk-sum of a
// blocked multiply (matrix/BlockMatrix.scala:177) is folded into ONE launch, so the fp32 accumulator never leaves registers.
struct SegMaps {
    CUtensorMap a[MAX_SEG];
    CUtensorMap b[MAX_SEG];
    int num_kb[MAX_SEG];
    int nseg;
};

struct Params {
    int M, N, K;
    void* C;
    long long ldc;
    int tiles_m, tiles_n;
    int c_is_f32;
    int accumulate;
};

__device__ __forceinline__ void tile_coords(int t, int tiles_m, int tiles_n, int& tm, int& tn) {
    const int band_tiles = BAND * tiles_n;
    const int band = t / band_tiles;
    const int r = t - band * band_tiles;
    const int rows_in_band = min(BAND, tiles_m - band * BAND);
    tn = r / rows_in_band;
    tm = band * BAND + (r - tn * rows_in_band);
}

template <bool TA, bool TB>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_bf16_wgmma_kernel(const __grid_constant__ SegMaps maps, const Params p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t bar_full = smem_base + NUM_STAGES * STAGE_BYTES;   // [NUM_STAGES]
    const uint32_t bar_empty = bar_full + 8 * NUM_STAGES;             // [NUM_STAGES]

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int num_tiles = p.tiles_m * p.tiles_n;
    int num_kb = 0;                     // k-slabs of all segments
    for (int sg = 0; sg < maps.nseg; ++sg) num_kb += maps.num_kb[sg];

    if (threadIdx.x == 0) {
        for (int s = 0; s < NUM_STAGES; ++s) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, NUM_CONSUMER_WARPS); }
        fence_barrier_init();
        tma_prefetch_desc(&maps.a[0]);
        tma_prefetch_desc(&maps.b[0]);
    }
    __syncthreads();

    if (warp < 4) {
        // ===================== TMA producer =====================
        setmaxnreg_dec<40>();
        if (warp == 0 && lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
                int tm, tn;
                tile_coords(t, p.tiles_m, p.tiles_n, tm, tn);
                const int m0 = tm * BM, n0 = tn * BN;
                for (int sg = 0; sg < maps.nseg; ++sg) {
                    const CUtensorMap* mapA = &maps.a[sg];
                    const CUtensorMap* mapB = &maps.b[sg];
                    const int nkb = maps.num_kb[sg];
                    for (int kb = 0; kb < nkb; ++kb) {
                        mbar_wait(bar_empty + 8 * stage, phase ^ 1);
                        const uint32_t full = bar_full + 8 * stage;
                        const uint32_t sA = smem_base + stage * STAGE_BYTES;
                        const uint32_t sB = sA + A_BYTES;
                        mbar_arrive_expect_tx(full, STAGE_BYTES);
                        const int k0 = kb * BK;
                        if (!TA) {
                            tma_load_2d(sA, mapA, full, m0, k0);
                            tma_load_2d(sA + 8192, mapA, full, m0 + 64, k0);
                        } else {
                            tma_load_2d(sA, mapA, full, k0, m0);
                        }
                        if (!TB) {
                            tma_load_2d(sB, mapB, full, k0, n0);
                        } else {
#pragma unroll
                            for (int b = 0; b < 4; ++b) tma_load_2d(sB + b * 8192, mapB, full, n0 + 64 * b, k0);
                        }
                        if (++stage == NUM_STAGES) { stage = 0; phase ^= 1; }
                    }
                }
            }
        }
        return;
    }

    // ===================== consumer warpgroups =====================
    setmaxnreg_inc<232>();
    const int wg = (warp >> 2) - 1;     // 0, 1: rows 64*wg .. 64*wg+63 of the tile
    const int wq = warp & 3;            // warp inside the warpgroup: accumulator rows 16*wq .. 16*wq+15
    int stage = 0;
    uint32_t phase = 0;
    float acc[128];
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        int tm, tn;
        tile_coords(t, p.tiles_m, p.tiles_n, tm, tn);
        int prev = -1;                  // stage read by the wgmma group still in flight
        for (int kb = 0; kb < num_kb; ++kb) {
            mbar_wait(bar_full + 8 * stage, phase);
            // both A layouts put this warpgroup's 64 rows 8 KiB into the stage
            const uint32_t sA = smem_base + stage * STAGE_BYTES + wg * 8192;
            const uint32_t sB = smem_base + stage * STAGE_BYTES + A_BYTES;
            wgmma_fence_operands(acc);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < BK / 16; ++k) {
                // MN-major: 16 k-rows of 128 B per k16 step; K-major: 32 B along the swizzled 128 B row
                const uint64_t adesc = !TA ? gmma_desc_sw128(sA + k * 2048, 8192, 1024) : gmma_desc_sw128(sA + k * 32, 0, 1024);
                const uint64_t bdesc = TB ? gmma_desc_sw128(sB + k * 2048, 8192, 1024) : gmma_desc_sw128(sB + k * 32, 0, 1024);
                wgmma_m64n256k16_bf16<!TA ? 1 : 0, TB ? 1 : 0>(acc, adesc, bdesc, (kb | k) ? 1u : 0u);
            }
            wgmma_commit();
            wgmma_wait<1>();            // keep this slab's group in flight; the previous slab's has retired
            if (prev >= 0) {
                __syncwarp();
                if (lane == 0) mbar_arrive(bar_empty + 8 * prev);  // this warp's reads of that stage are done
            }
            prev = stage;
            if (++stage == NUM_STAGES) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        wgmma_fence_operands(acc);
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty + 8 * prev);

        // ---- epilogue: accumulator fragment -> C.  acc[4j + 2h + e] is row 16*wq + lane/4 + 8h, column 8j + 2*(lane%4) + e
        const int mrow = tm * BM + wg * 64 + wq * 16 + (lane >> 2);
        const int ncol = tn * BN + 2 * (lane & 3);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int m = mrow + 8 * h;
            if (m >= p.M) continue;
            if (p.c_is_f32) {
                float* crow = static_cast<float*>(p.C) + m;
#pragma unroll
                for (int jc = 0; jc < 32; jc += 8) {
                    float old[16];
                    if (p.accumulate) {  // 16 loads first: one memory latency per 16 values, not 16 dependent ones
#pragma unroll
                        for (int j = 0; j < 8; ++j)
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                const int n = ncol + 8 * (jc + j) + e;
                                old[2 * j + e] = (n < p.N) ? __ldcg(crow + (long long)n * p.ldc) : 0.f;
                            }
                    }
#pragma unroll
                    for (int j = 0; j < 8; ++j)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int n = ncol + 8 * (jc + j) + e;
                            if (n < p.N) {
                                float x = acc[4 * (jc + j) + 2 * h + e];
                                if (p.accumulate) x += old[2 * j + e];
                                crow[(long long)n * p.ldc] = x;
                            }
                        }
                }
            } else {
                __nv_bfloat16* crow = static_cast<__nv_bfloat16*>(p.C) + m;
#pragma unroll
                for (int j = 0; j < 32; ++j)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int n = ncol + 8 * j + e;
                        if (n < p.N) {
                            float x = acc[4 * j + 2 * h + e];
                            __nv_bfloat16* dst = crow + (long long)n * p.ldc;
                            if (p.accumulate) x += __bfloat162float(*dst);
                            *dst = __float2bfloat16_rn(x);
                        }
                    }
            }
        }
    }
}

}  // namespace

cudaError_t gemm_bf16_segments(bool transA, bool transB, int M, int N, int nseg, const int* Kseg, const void* const* A,
                               const long long* lda, const void* const* B, const long long* ldb, void* C, long long ldc,
                               bool c_is_f32, bool accumulate, int num_sms, cudaStream_t stream) {
    if (M <= 0 || N <= 0) return cudaSuccess;
    if (nseg <= 0 || nseg > MAX_SEG || !tma_encode_fn()) return cudaErrorNotSupported;
    static thread_local SegMaps maps;
    maps.nseg = nseg;
    int Ktot = 0;
    for (int sg = 0; sg < nseg; ++sg) {
        const int K = Kseg[sg];
        if (K <= 0) return cudaErrorNotSupported;
        const bool aligned = ((reinterpret_cast<uintptr_t>(A[sg]) | reinterpret_cast<uintptr_t>(B[sg])) & 15) == 0 &&
                             (lda[sg] % 8 == 0) && (ldb[sg] % 8 == 0);
        if (!aligned) return cudaErrorNotSupported;
        constexpr CUtensorMapDataType BF16 = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
        const bool ok = (!transA ? tma_map(&maps.a[sg], BF16, A[sg], M, K, lda[sg] * 2, 64, 64)
                                 : tma_map(&maps.a[sg], BF16, A[sg], K, M, lda[sg] * 2, 64, 128)) &&
                        (!transB ? tma_map(&maps.b[sg], BF16, B[sg], K, N, ldb[sg] * 2, 64, 256)
                                 : tma_map(&maps.b[sg], BF16, B[sg], N, K, ldb[sg] * 2, 64, 64));
        if (!ok) return cudaErrorNotSupported;
        maps.num_kb[sg] = (K + BK - 1) / BK;
        Ktot += K;
    }
    Params p;
    p.M = M; p.N = N; p.K = Ktot; p.C = C; p.ldc = ldc;
    p.tiles_m = (M + BM - 1) / BM;
    p.tiles_n = (N + BN - 1) / BN;
    p.c_is_f32 = c_is_f32 ? 1 : 0;
    p.accumulate = accumulate ? 1 : 0;
    const int grid = min(p.tiles_m * p.tiles_n, num_sms);
    if (!transA && !transB) return launch_with_smem<gemm_bf16_wgmma_kernel<false, false>>(grid, NUM_THREADS, SMEM_BYTES, stream, maps, p);
    if (transA && !transB) return launch_with_smem<gemm_bf16_wgmma_kernel<true, false>>(grid, NUM_THREADS, SMEM_BYTES, stream, maps, p);
    if (!transA && transB) return launch_with_smem<gemm_bf16_wgmma_kernel<false, true>>(grid, NUM_THREADS, SMEM_BYTES, stream, maps, p);
    return launch_with_smem<gemm_bf16_wgmma_kernel<true, true>>(grid, NUM_THREADS, SMEM_BYTES, stream, maps, p);
}

}  // namespace mb

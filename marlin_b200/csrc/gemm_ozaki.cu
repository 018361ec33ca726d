// fp64 block GEMM on the int8 tensor cores (wgmma.mma_async .s32.s8.s8).
//
// The fp64 tensor-core rate (DMMA) is a small fraction of the int8 rate.  This path splits
// each operand into `s` signed 7-bit digit planes after exact power-of-two row/column scaling (an Ozaki split):
//     a_ik = 2^(eA_i - P) * X_ik,   X_ik = sum_t dA_t(i,k) * 128^(s-t),   |dA_t| <= 64,   P = 7s - 1
//     b_kj = 2^(eB_j - P) * Y_kj    likewise
// so that   sum_k a_ik b_kj = 2^(eA_i + eB_j - 2P) * sum_{t,u} 128^(2s-t-u) * [ sum_k dA_t(i,k) dB_u(k,j) ] .
// Every bracket is an int8 GEMM accumulated EXACTLY in int32 registers.  Pairs with t + u > s + 1 are dropped (their
// weight is below the rounding of the operands), the brackets of one group d = t + u share an accumulator, and the
// epilogue adds the groups into C in fp64 from the least significant group up.  With s = 7 the result is within a few
// 1e-14 of the exact product relative to (|A||B|)_ij for well-scaled rows; s = 6 stays below 1e-11.
// The error is relative to rowmax_i(A)*colmax_j(B)*K, not to (|A||B|)_ij, so this mode is opt-in (mb_set_fp64_mode)
// and the DMMA kernel remains the default.
//
// Kernel structure = the bf16 wgmma kernel (a TMA producer warpgroup, two consumer warpgroups of 64 rows each that hold
// a 64 x 256 int32 accumulator in registers), with 3-D TMA maps over the digit planes.  wgmma takes 8-bit operands
// K-major only, so both digit planes are stored k-contiguous: A planes [m][k], B planes [n][k].  After the last
// bracket of a group the consumers fold the accumulator into C with an fp64 read-modify-write.
#include "gemm_ozaki.h"
#include "ptx.cuh"
#include "launch.h"
#include "tma.h"

namespace mb {

namespace {

constexpr int BM = 128, BN = 256, BK = 128;       // BK int8 = 128 B = one swizzle row
constexpr int A_BYTES = BM * BK;                   // 16 KiB
constexpr int B_BYTES = BN * BK;                   // 32 KiB
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int NUM_STAGES = 4;
constexpr int NUM_CONSUMER_WARPS = 8;
constexpr int NUM_THREADS = 128 + NUM_CONSUMER_WARPS * 32;
constexpr int SMEM_BYTES = NUM_STAGES * STAGE_BYTES + 1024 + 256;
constexpr int BAND = 16;

struct Params {
    int M, N, K, s;
    int bits;          // digit width: 7 (|digit| <= 64) or 8 (|digit| <= 128, top digit <= 64)
    int P;             // fractional bits of the scaled operands: bits*s - (bits == 8 ? 2 : 1)
    double* C;
    long long ldc;
    const int* eA;
    const int* eB;
    int tiles_m, tiles_n;
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

__device__ __forceinline__ void tma_load_3d(uint32_t dst_smem, const CUtensorMap* map, uint32_t bar, int32_t c0, int32_t c1,
                                            int32_t c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(dst_smem), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}

// 2^ex exactly as ldexp(1.0, ex), without the library call (a call inside the consumer loop spills the accumulator)
__device__ __forceinline__ double pow2_scale(int ex) {
    if (ex >= -1022 && ex <= 1023) return __hiloint2double((ex + 1023) << 20, 0);
    if (ex > 1023) return __longlong_as_double(0x7FF0000000000000ll);      // overflow: +inf
    if (ex >= -1074) return __longlong_as_double(1ll << (ex + 1074));      // subnormal
    return 0.0;
}

__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_ozaki_i8_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, const Params p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t bar_full = smem_base + NUM_STAGES * STAGE_BYTES;
    const uint32_t bar_empty = bar_full + 8 * NUM_STAGES;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int num_tiles = p.tiles_m * p.tiles_n;
    const int num_kb = (p.K + BK - 1) / BK;
    const int s = p.s;

    if (threadIdx.x == 0) {
        for (int i = 0; i < NUM_STAGES; ++i) { mbar_init(bar_full + 8 * i, 1); mbar_init(bar_empty + 8 * i, NUM_CONSUMER_WARPS); }
        fence_barrier_init();
        tma_prefetch_desc(&mapA);
        tma_prefetch_desc(&mapB);
    }
    __syncthreads();

    if (warp < 4) {
        setmaxnreg_dec<40>();
        if (warp == 0 && lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
                int tm, tn;
                tile_coords(t, p.tiles_m, p.tiles_n, tm, tn);
                const int m0 = tm * BM, n0 = tn * BN;
                for (int d = s + 1; d >= 2; --d) {
                    const int t_lo = max(1, d - s), t_hi = min(s, d - 1);
                    for (int ta = t_lo; ta <= t_hi; ++ta) {
                        const int ub = d - ta;
                        for (int kb = 0; kb < num_kb; ++kb) {
                            mbar_wait(bar_empty + 8 * stage, phase ^ 1);
                            const uint32_t full = bar_full + 8 * stage;
                            const uint32_t sA = smem_base + stage * STAGE_BYTES;
                            mbar_arrive_expect_tx(full, STAGE_BYTES);
                            tma_load_3d(sA, &mapA, full, kb * BK, m0, ta - 1);
                            tma_load_3d(sA + A_BYTES, &mapB, full, kb * BK, n0, ub - 1);
                            if (++stage == NUM_STAGES) { stage = 0; phase ^= 1; }
                        }
                    }
                }
            }
        }
        return;
    }

    setmaxnreg_inc<232>();
    const int wg = (warp >> 2) - 1;     // 0, 1: rows 64*wg .. 64*wg+63 of the tile
    const int wq = warp & 3;            // accumulator rows 16*wq .. 16*wq+15 of the warpgroup's 64
    const int P2 = 2 * p.P;
    int stage = 0;
    uint32_t phase = 0;
    int32_t acc[128];
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        int tm, tn;
        tile_coords(t, p.tiles_m, p.tiles_n, tm, tn);
        // acc[4j + 2h + e] is row mrow + 8h, column ncol + 8j + e
        const int mrow = tm * BM + wg * 64 + wq * 16 + (lane >> 2);
        const int ncol = tn * BN + 2 * (lane & 3);
        int ea[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) ea[h] = (mrow + 8 * h < p.M) ? __ldg(p.eA + mrow + 8 * h) : 0;
        for (int d = s + 1; d >= 2; --d) {
            const int npairs = min(s, d - 1) - max(1, d - s) + 1;
            uint32_t first = 1;
            int prev = -1;              // stage read by the wgmma group still in flight
            for (int pr = 0; pr < npairs; ++pr) {
                for (int kb = 0; kb < num_kb; ++kb) {
                    mbar_wait(bar_full + 8 * stage, phase);
                    const uint32_t sA = smem_base + stage * STAGE_BYTES + wg * 8192;
                    const uint32_t sB = smem_base + stage * STAGE_BYTES + A_BYTES;
                    wgmma_fence_operands(acc);
                    wgmma_fence();
#pragma unroll
                    for (int k = 0; k < BK / 32; ++k) {
                        // both planes K-major: 32 B along the swizzled 128 B row per k32 step
                        wgmma_m64n256k32_s8(acc, gmma_desc_sw128(sA + k * 32, 0, 1024), gmma_desc_sw128(sB + k * 32, 0, 1024),
                                            first ? 0u : 1u);
                        first = 0;
                    }
                    wgmma_commit();
                    wgmma_wait<1>();    // keep this slab's group in flight; the previous slab's has retired
                    if (prev >= 0) {
                        __syncwarp();
                        if (lane == 0) mbar_arrive(bar_empty + 8 * prev);
                    }
                    prev = stage;
                    if (++stage == NUM_STAGES) { stage = 0; phase ^= 1; }
                }
            }
            wgmma_wait<0>();
            wgmma_fence_operands(acc);
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_empty + 8 * prev);
            // fold group d: C (+)= acc * 2^(ex_m + eB[n]); 8 old values of C are loaded before any store so the
            // read-modify-write costs one memory latency per 8 values instead of 8 dependent ones
            const bool init = (d == s + 1) && !p.accumulate;
            // opaque copy: keeps the compiler from hoisting the 64 column addresses and eB loads out of the d loop,
            // which would not fit in registers next to the accumulator
            int nc = ncol;
            asm volatile("" : "+r"(nc));
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = mrow + 8 * h;
                if (m >= p.M) continue;
                const int ex_m = ea[h] - P2 + p.bits * (2 * s - d);
                double* crow = p.C + m;
#pragma unroll
                for (int jc = 0; jc < 32; jc += 4) {
                    double old[8];
                    if (!init) {
#pragma unroll
                        for (int j = 0; j < 4; ++j)
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                const int n = nc + 8 * (jc + j) + e;
                                old[2 * j + e] = (n < p.N) ? __ldcg(crow + (long long)n * p.ldc) : 0.0;
                            }
                    }
#pragma unroll
                    for (int j = 0; j < 4; ++j)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int n = nc + 8 * (jc + j) + e;
                            if (n < p.N) {
                                // a zero group adds +0 without forming 2^ex, which overflows to +Inf for the low groups
                                // of rows / columns near DBL_MAX (0 * Inf = NaN) and is meaningless for the sentinel
                                // exponent of a non-finite row / column
                                const int32_t av = acc[4 * (jc + j) + 2 * h + e];
                                const double term = av != 0 ? (double)av * pow2_scale(ex_m + __ldg(p.eB + n)) : 0.0;
                                crow[(long long)n * p.ldc] = init ? term : (old[2 * j + e] + term);
                            }
                        }
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------- operand splitting
// Row / column maxima are taken over the bit patterns of |a|: non-negative doubles order like their bit patterns, and
// +Inf and every NaN (sign cleared) lie above all finite values, so a non-finite entry always shows in its maximum (fmax
// would drop a NaN).  Such a row / column gets the exponent NONFINITE_EXP and zero digits, so it adds nothing to the
// int8 products, and ozaki_fixup_kernel recomputes its entries of C in plain fp64.
constexpr unsigned long long INF_BITS = 0x7FF0000000000000ull;
constexpr int NONFINITE_EXP = 1 << 20;

__device__ __forceinline__ unsigned long long abs_bits(double a) {
    return (unsigned long long)__double_as_longlong(a) & 0x7FFFFFFFFFFFFFFFull;
}

__global__ void ozaki_rowmax_kernel(const double* __restrict__ A, long long lda, int M, int K, int kchunk,
                                    unsigned long long* __restrict__ rowmax_bits) {
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= M) return;
    const int k0 = blockIdx.y * kchunk, k1 = min(K, k0 + kchunk);
    unsigned long long r = 0;
    for (int k = k0; k < k1; ++k) r = max(r, abs_bits(A[m + (long long)k * lda]));
    atomicMax(rowmax_bits + m, r);
}

__device__ __forceinline__ int scale_exponent(unsigned long long rbits) {
    // smallest e with r < 2^e (r > 0); 0 for an all-zero row/column; NONFINITE_EXP for a row/column holding NaN or Inf
    if (rbits >= INF_BITS) return NONFINITE_EXP;
    const double r = __longlong_as_double((long long)rbits);
    if (!(r > 0.0)) return 0;
    return ilogb(r) + 1;
}

// digits of X = rint(a * 2^(P - e)), most significant first: out[t] for t = 0..s-1, each in [-64, 64]; all zero for a
// non-finite row / column, which the fix-up pass recomputes
__device__ __forceinline__ void split_digits(double a, int e, int s, int bits, int P, signed char* digs) {
    if (e == NONFINITE_EXP) {
        for (int t = 0; t < s; ++t) digs[t] = 0;
        return;
    }
    long long X = __double2ll_rn(ldexp(a, P - e));
    const long long half = 1ll << (bits - 1), mask = (1ll << bits) - 1;
    for (int t = s - 1; t >= 1; --t) {
        const long long dgt = ((X + half) & mask) - half;
        digs[t] = (signed char)dgt;
        X = (X - dgt) >> bits;
    }
    digs[0] = (signed char)X;          // |X| <= 64 by the choice of P
}

// A (M x K, column-major) -> planes A8[t][m * ld8 + k] (k contiguous, as wgmma wants 8-bit operands).  Reads stay
// coalesced along m; each thread packs the digits of 8 consecutive k into one 8-byte store per plane.
__global__ void ozaki_split_a_kernel(const double* __restrict__ A, long long lda, int M, int K, int s, int bits, int P,
                                     const unsigned long long* __restrict__ rowmax_bits, signed char* __restrict__ A8,
                                     long long ld8, long long plane, int* __restrict__ eA) {
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= M) return;
    const int e = scale_exponent(rowmax_bits[m]);
    if (blockIdx.y == 0) eA[m] = e;
    const int kchunk = ((K + gridDim.y - 1) / gridDim.y + 7) & ~7;
    const int k0 = blockIdx.y * kchunk, k1 = min(K, k0 + kchunk);
    signed char digs[8];
    for (int k = k0; k < k1; k += 8) {
        unsigned long long packed[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (int i = 0; i < 8 && k + i < k1; ++i) {
            split_digits(A[m + (long long)(k + i) * lda], e, s, bits, P, digs);
#pragma unroll
            for (int t = 0; t < 8; ++t)
                if (t < s) packed[t] |= (unsigned long long)(unsigned char)digs[t] << (8 * i);
        }
        // k is a multiple of 8 and ld8 of 16, and k + 8 <= ld8: an aligned store inside the row (zeros past K)
#pragma unroll
        for (int t = 0; t < 8; ++t)
            if (t < s) *reinterpret_cast<unsigned long long*>(A8 + t * plane + (long long)m * ld8 + k) = packed[t];
    }
}

// B (K x N, column-major): one block per column -> planes B8[u][j * ld8 + k] (k contiguous)
__global__ void __launch_bounds__(256) ozaki_split_b_kernel(const double* __restrict__ B, long long ldb, int K, int N, int s,
                                                           int bits, int P,
                                                           signed char* __restrict__ B8, long long ld8, long long plane,
                                                           int* __restrict__ eB) {
    __shared__ unsigned long long red[8];
    const int j = blockIdx.x;
    const double* col = B + (long long)j * ldb;
    unsigned long long r = 0;
    for (int k = threadIdx.x; k < K; k += 256) r = max(r, abs_bits(col[k]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) r = max(r, __shfl_xor_sync(0xffffffffu, r, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = r;
    __syncthreads();
    r = red[0];
#pragma unroll
    for (int w = 1; w < 8; ++w) r = max(r, red[w]);
    const int e = scale_exponent(r);
    if (threadIdx.x == 0) eB[j] = e;
    signed char digs[8];
    for (int k = threadIdx.x; k < K; k += 256) {
        split_digits(col[k], e, s, bits, P, digs);
        for (int t = 0; t < s; ++t) B8[t * plane + (long long)j * ld8 + k] = digs[t];
    }
}

// C(i, j) (+)= sum_k A(i, k) B(k, j) in fp64, k ascending, for every i whose row of A or j whose column of B holds a NaN
// or Inf (eA / eB == NONFINITE_EXP): the IEEE result the DMMA kernel gives, instead of the digits' finite nonsense.
// Blocks 0..M-1 take row i, blocks M..M+N-1 column j (skipping flagged rows, done by their row block); a block whose
// row / column is finite exits at once, so the pass costs one tiny launch when nothing is flagged.
__global__ void __launch_bounds__(128) ozaki_fixup_kernel(const double* __restrict__ A, long long lda, const double* __restrict__ B,
                                                          long long ldb, double* __restrict__ C, long long ldc, int M, int N,
                                                          int K, int accumulate, const int* __restrict__ eA,
                                                          const int* __restrict__ eB) {
    const bool row = blockIdx.x < (unsigned)M;
    const int idx = row ? blockIdx.x : blockIdx.x - M;
    if ((row ? eA[idx] : eB[idx]) != NONFINITE_EXP) return;
    const int count = row ? N : M;
    for (int o = threadIdx.x; o < count; o += blockDim.x) {
        const int i = row ? idx : o, j = row ? o : idx;
        if (!row && eA[i] == NONFINITE_EXP) continue;
        double s = 0.0;
        for (int k = 0; k < K; ++k) s = __dadd_rn(s, __dmul_rn(A[i + (long long)k * lda], B[k + (long long)j * ldb]));
        double* c = C + i + (long long)j * ldc;
        *c = accumulate ? __dadd_rn(*c, s) : s;
    }
}

inline size_t round_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

}  // namespace

size_t ozaki_workspace_bytes(int M, int N, int K, int s) {
    const size_t ldA = round_up((size_t)K, 16), ldB = round_up((size_t)K, 16);
    return round_up(ldA * M * s, 256) + round_up(ldB * N * s, 256) + round_up((size_t)M * 8, 256) + round_up((size_t)M * 4, 256) +
           round_up((size_t)N * 4, 256);
}

bool ozaki_supported(int M, int N, int K, int s, int bits) {
    // int32 accumulation of up to s pairs of K products of magnitude <= 2^(2*(bits-1)) must stay below 2^31
    return s >= 2 && s <= 8 && (bits == 7 || bits == 8) && M > 0 && N > 0 && K > 0 &&
           (long long)K * s * (1ll << (2 * (bits - 1))) < (1ll << 31) && tma_encode_fn() != nullptr;
}

cudaError_t gemm_f64_ozaki(int M, int N, int K, const double* A, long long lda, const double* B, long long ldb, double* C,
                           long long ldc, bool accumulate, int s, int bits, void* workspace, int num_sms, cudaStream_t stream) {
    if (!ozaki_supported(M, N, K, s, bits)) return cudaErrorNotSupported;
    const int P = bits * s - (bits == 8 ? 2 : 1);
    const size_t ldA = round_up((size_t)K, 16), ldB = round_up((size_t)K, 16);
    const size_t planeA = ldA * M, planeB = ldB * N;
    char* w = static_cast<char*>(workspace);
    signed char* A8 = reinterpret_cast<signed char*>(w);
    w += round_up(planeA * s, 256);
    signed char* B8 = reinterpret_cast<signed char*>(w);
    w += round_up(planeB * s, 256);
    unsigned long long* rowmax = reinterpret_cast<unsigned long long*>(w);
    w += round_up((size_t)M * 8, 256);
    int* eA = reinterpret_cast<int*>(w);
    w += round_up((size_t)M * 4, 256);
    int* eB = reinterpret_cast<int*>(w);

    cudaError_t e = cudaMemsetAsync(rowmax, 0, (size_t)M * 8, stream);
    if (e != cudaSuccess) return e;
    const int ksplit = max(1, min(64, K / 256));
    const int kchunk = (K + ksplit - 1) / ksplit;
    dim3 grid_a((M + 127) / 128, ksplit);
    ozaki_rowmax_kernel<<<grid_a, 128, 0, stream>>>(A, lda, M, K, kchunk, rowmax);
    if ((e = launched()) != cudaSuccess) return e;
    ozaki_split_a_kernel<<<grid_a, 128, 0, stream>>>(A, lda, M, K, s, bits, P, rowmax, A8, (long long)ldA, (long long)planeA, eA);
    if ((e = launched()) != cudaSuccess) return e;
    ozaki_split_b_kernel<<<N, 256, 0, stream>>>(B, ldb, K, N, s, bits, P, B8, (long long)ldB, (long long)planeB, eB);
    if ((e = launched()) != cudaSuccess) return e;

    CUtensorMap mA, mB;
    if (!tma_map_3d(&mA, CU_TENSOR_MAP_DATA_TYPE_UINT8, A8, K, M, s, ldA, planeA, 128, 128)) return cudaErrorNotSupported;
    if (!tma_map_3d(&mB, CU_TENSOR_MAP_DATA_TYPE_UINT8, B8, K, N, s, ldB, planeB, 128, 256)) return cudaErrorNotSupported;
    Params p;
    p.M = M; p.N = N; p.K = K; p.s = s; p.bits = bits; p.P = P; p.C = C; p.ldc = ldc; p.eA = eA; p.eB = eB;
    p.tiles_m = (M + BM - 1) / BM;
    p.tiles_n = (N + BN - 1) / BN;
    p.accumulate = accumulate ? 1 : 0;
    e = launch_with_smem<gemm_ozaki_i8_kernel>(min(p.tiles_m * p.tiles_n, num_sms), NUM_THREADS, SMEM_BYTES, stream, mA, mB, p);
    if (e != cudaSuccess) return e;
    // stream-ordered after the int8 kernel, which leaves the flagged entries of C as they were (accumulate) or +0
    ozaki_fixup_kernel<<<M + N, 128, 0, stream>>>(A, lda, B, ldb, C, ldc, M, N, K, p.accumulate, eA, eB);
    return launched();
}

}  // namespace mb

// fp64 block GEMM for sm_90a — replaces SubMatrix.multiply -> Breeze `*` -> netlib dgemm
// (reference: matrix/SubMatrix.scala:87-91; inline twins matrix/DenseVecMatrix.scala:122,129,1676).
//
// wgmma has no fp64 type, so the fp64 tensor-core path on H100 is
// DMMA (mma.sync.m8n8k4.f64 -> SASS DMMA.8x8x4).  Design:
//   * persistent CTAs (one per SM), 128x128 C tile per CTA, accumulators in registers
//     (8 consumer warps x 64x32 warp tile = 64 doubles / thread);
//   * a dedicated producer warp streams A/B k-slabs (BK = 16) through a 6-stage shared-memory
//     ring with TMA (cp.async.bulk.tensor.2d, SWIZZLE_128B) + mbarrier full/empty pairs;
//     TMA zero-fills out-of-range rows/cols, so ragged blocks (ceil-sized last block of
//     BlockMatrix, matrix/BlockMatrix.scala:73-74) need no host-side padding;
//   * operand fragments are read with conflict-free 128-bit LDS from the swizzled tiles: the
//     MMA row/col and k slots are permuted (any permutation of the m, n, k index sets is a valid
//     GEMM as long as A, B and C agree) so that every quarter-warp hits 8 distinct 16B chunks;
//   * setmaxnreg moves registers from the producer warpgroup to the two consumer warpgroups.
//
// Both operands may be 'N' or 'T' (Breeze isTranspose views): an operand whose contiguous
// dimension is M/N ("MN form") is staged as 8 boxes of [16 k-rows][16 mn] and one whose
// contiguous dimension is K ("K form") as one box of [128 mn-rows][16 k].
#include "gemm_f64.h"
#include "ptx.cuh"
#include <atomic>
#include <cstdlib>

namespace mb {

namespace {

constexpr int BM = 128, BN = 128, BK = 16;
constexpr int OPERAND_BYTES = BM * BK * 8;          // 16 KiB per operand per stage
constexpr int STAGE_BYTES = 2 * OPERAND_BYTES;      // 32 KiB
constexpr int NUM_STAGES = 6;                       // 192 KiB ring
constexpr int NUM_CONSUMER_WARPS = 8;
constexpr int NUM_THREADS = 128 + NUM_CONSUMER_WARPS * 32;   // producer warpgroup + 2 consumer warpgroups
constexpr int SMEM_BYTES = NUM_STAGES * STAGE_BYTES + 2 * NUM_STAGES * 8 + 1024;
constexpr int BAND = 16;                            // tile-rows per rasterisation band (L2 reuse)

struct Params {
    int M, N, K;
    double alpha, beta;
    double* C;
    long long ldc;
    int tiles_m, tiles_n;
};

__device__ __forceinline__ int perm8(int r) { return ((r & 1) << 2) | (r >> 1); }

// tile id -> (tile_m, tile_n): bands of BAND tile-rows, column-major inside a band, so the ~132
// tiles in flight cover a BAND x (132/BAND) patch and share A row-panels / B column-panels in L2.
__device__ __forceinline__ void tile_coords(int t, int tiles_m, int tiles_n, int& tm, int& tn) {
    const int band_tiles = BAND * tiles_n;
    const int band = t / band_tiles;
    const int r = t - band * band_tiles;
    const int rows_in_band = min(BAND, tiles_m - band * BAND);
    tn = r / rows_in_band;
    tm = band * BAND + (r - tn * rows_in_band);
}

// Split-K schedule of the Gramian (syrk_f64_dmma_kernel): work item w = split * tri_tiles + t covers lower-triangle tile t
// (tm >= tn, row-major over the triangle) for k in [split * kchunk, min(K, (split + 1) * kchunk)) and stores its partial
// tile at C + split * split_stride.
struct SyrkSched {
    int splits, tri_tiles, kchunk;
    long long split_stride;
};

__device__ __forceinline__ void tri_coords(int t, int& tm, int& tn) {
    int r = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
    while ((r + 1) * (r + 2) / 2 <= t) ++r;
    while (r * (r + 1) / 2 > t) --r;
    tm = r;
    tn = t - r * (r + 1) / 2;
}

// The persistent TMA + DMMA mainloop shared by the GEMM (SYRK = false: every tile of C, the whole K range, C = alpha*acc +
// beta*C) and the Gramian (SYRK = true: lower-triangle tiles only, split-K partials stored to a workspace).
template <bool TA, bool TB, bool SYRK>
__device__ __forceinline__ void dmma_persistent(const CUtensorMap& mapA, const CUtensorMap& mapB, const Params& p,
                                                const SyrkSched& sk) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t bar_full = smem_base + NUM_STAGES * STAGE_BYTES;
    const uint32_t bar_empty = bar_full + NUM_STAGES * 8;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int num_tiles = SYRK ? sk.tri_tiles * sk.splits : p.tiles_m * p.tiles_n;
    const int num_kb = (p.K + BK - 1) / BK;

    if (threadIdx.x == 0) {
        for (int s = 0; s < NUM_STAGES; ++s) {
            mbar_init(bar_full + 8 * s, 1);
            mbar_init(bar_empty + 8 * s, NUM_CONSUMER_WARPS);
        }
        fence_barrier_init();
        tma_prefetch_desc(&mapA);
        tma_prefetch_desc(&mapB);
    }
    __syncthreads();

    if (warp < 4) {
        // ===================== producer warpgroup =====================
        setmaxnreg_dec<40>();
        if (warp == 0 && lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
                int tm, tn, kb_begin = 0, kb_end = num_kb;
                if constexpr (SYRK) {
                    const int split = t / sk.tri_tiles;
                    tri_coords(t - split * sk.tri_tiles, tm, tn);
                    kb_begin = split * (sk.kchunk / BK);
                    kb_end = min(num_kb, kb_begin + sk.kchunk / BK);
                } else {
                    tile_coords(t, p.tiles_m, p.tiles_n, tm, tn);
                }
                const int m0 = tm * BM, n0 = tn * BN;
                for (int kb = kb_begin; kb < kb_end; ++kb) {
                    mbar_wait(bar_empty + 8 * stage, phase ^ 1);
                    const uint32_t full = bar_full + 8 * stage;
                    const uint32_t sA = smem_base + stage * STAGE_BYTES;
                    const uint32_t sB = sA + OPERAND_BYTES;
                    mbar_arrive_expect_tx(full, STAGE_BYTES);
                    const int k0 = kb * BK;
                    if (!TA) {
#pragma unroll
                        for (int b = 0; b < 8; ++b) tma_load_2d(sA + b * 2048, &mapA, full, m0 + 16 * b, k0);
                    } else {
                        tma_load_2d(sA, &mapA, full, k0, m0);
                    }
                    if (!TB) {
                        tma_load_2d(sB, &mapB, full, k0, n0);
                    } else {
#pragma unroll
                        for (int b = 0; b < 8; ++b) tma_load_2d(sB + b * 2048, &mapB, full, n0 + 16 * b, k0);
                    }
                    if (++stage == NUM_STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
        return;
    }

    // ========================= consumer warpgroups =========================
    setmaxnreg_inc<232>();
    const int cw = warp - 4;          // 0..7
    const int warp_m = cw & 1;        // 64-row slab
    const int warp_n = cw >> 1;       // 32-col slab
    const int r = lane >> 2;          // MMA row (A) / col (B) index of this lane
    const int q = lane & 3;           // MMA k slot of this lane
    const int pr = perm8(r);

    // Per-lane byte offsets of the fragment loads inside one operand tile (see header comment).
    //  MN form: box t' (16 mn x 16 k, 2 KiB), k-row = 8h + 2q + p, 16B chunk = r ^ ((2q+p)&7)
    //           -> doubles (mn = 16t' + 2r, 16t' + 2r + 1)  = MMA tiles 2t', 2t'+1, row r.
    //  K  form: row mn = base + 8u + perm8(r), 16B chunk = (4h + q) ^ perm8(r)
    //           -> doubles (k = 8h + 2q, 8h + 2q + 1)       = phases p = 0, 1.
    uint32_t offA[2][2], offB[2][2];   // [h][p] for MN form, [h][0] used for K form
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int pp = 0; pp < 2; ++pp) {
            const int krow = 8 * h + 2 * q + pp;
            const uint32_t mn_off = krow * 128 + ((r ^ (krow & 7)) << 4);
            const uint32_t k_off = pr * 128 + ((((4 * h + q) ^ pr) & 7) << 4);
            offA[h][pp] = !TA ? (warp_m * 4 * 2048 + mn_off) : (warp_m * 64 * 128 + k_off);
            offB[h][pp] = TB ? (warp_n * 2 * 2048 + mn_off) : (warp_n * 32 * 128 + k_off);
        }
    }

    int stage = 0;
    uint32_t phase = 0;
    const bool vec_ok = ((reinterpret_cast<uintptr_t>(p.C) & 15) == 0) && ((p.ldc & 1) == 0);

    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        int tm_, tn_, k_begin = 0, k_end = p.K;
        double* Cout = p.C;
        if constexpr (SYRK) {
            const int split = t / sk.tri_tiles;
            tri_coords(t - split * sk.tri_tiles, tm_, tn_);
            k_begin = split * sk.kchunk;
            k_end = min(p.K, k_begin + sk.kchunk);
            Cout = p.C + split * sk.split_stride;
        } else {
            tile_coords(t, p.tiles_m, p.tiles_n, tm_, tn_);
        }
        const int m0 = tm_ * BM, n0 = tn_ * BN;

        double acc[8][4][2];
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;

        // bounded by p.K (a kernel parameter) rather than num_kb: one register fewer, which the <N,T> instance needs
        // to fit sm_90a's 168-register budget without a spill
        for (int k0 = k_begin; k0 < k_end; k0 += BK) {
            mbar_wait(bar_full + 8 * stage, phase);
            const uint32_t sA = smem_base + stage * STAGE_BYTES;
            const uint32_t sB = sA + OPERAND_BYTES;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                double a[8][2];   // [m-tile][phase]
                double b[4][2];   // [n-tile][phase]
                if (!TA) {
#pragma unroll
                    for (int tp = 0; tp < 4; ++tp)
#pragma unroll
                        for (int pp = 0; pp < 2; ++pp)
                            lds128(a[2 * tp][pp], a[2 * tp + 1][pp], sA + offA[h][pp] + tp * 2048);
                } else {
#pragma unroll
                    for (int u = 0; u < 8; ++u) lds128(a[u][0], a[u][1], sA + offA[h][0] + u * 8 * 128);
                }
                if (!TB) {
#pragma unroll
                    for (int u = 0; u < 4; ++u) lds128(b[u][0], b[u][1], sB + offB[h][0] + u * 8 * 128);
                } else {
#pragma unroll
                    for (int tp = 0; tp < 2; ++tp)
#pragma unroll
                        for (int pp = 0; pp < 2; ++pp)
                            lds128(b[2 * tp][pp], b[2 * tp + 1][pp], sB + offB[h][pp] + tp * 2048);
                }
                if (h == 1) {
                    // all reads of this stage are issued; hand the slot back to the producer
                    __syncwarp();
                    if (lane == 0) mbar_arrive(bar_empty + 8 * stage);
                }
#pragma unroll
                for (int pp = 0; pp < 2; ++pp)
#pragma unroll
                    for (int i = 0; i < 8; ++i)
#pragma unroll
                        for (int j = 0; j < 4; ++j) dmma_m8n8k4(acc[i][j][0], acc[i][j][1], a[i][pp], b[j][pp]);
            }
            if (++stage == NUM_STAGES) { stage = 0; phase ^= 1; }
        }

        // ---------------- epilogue: C = alpha*acc + beta*C ----------------
        // lane holds C[mrow(i-tile, r)][ncol(j-tile, 2q + jj)]
        const double alpha = p.alpha, beta = p.beta;
        const bool use_beta = (beta != 0.0);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
#pragma unroll
            for (int jj = 0; jj < 2; ++jj) {
                const int cj = 2 * q + jj;
                const int n = n0 + warp_n * 32 + (!TB ? (8 * j + perm8(cj)) : (16 * (j >> 1) + 2 * cj + (j & 1)));
                if (n >= p.N) continue;
                double* ccol = Cout + (long long)n * p.ldc;
                if (!TA) {
#pragma unroll
                    for (int tp = 0; tp < 4; ++tp) {
                        const int m = m0 + warp_m * 64 + 16 * tp + 2 * r;
                        if (m >= p.M) continue;
                        double v0 = alpha * acc[2 * tp][j][jj];
                        double v1 = alpha * acc[2 * tp + 1][j][jj];
                        if (vec_ok && m + 1 < p.M) {
                            double2* ptr = reinterpret_cast<double2*>(ccol + m);
                            if (use_beta) {
                                const double2 old = *ptr;
                                v0 += beta * old.x;
                                v1 += beta * old.y;
                            }
                            *ptr = make_double2(v0, v1);
                        } else {
                            if (use_beta) v0 += beta * ccol[m];
                            ccol[m] = v0;
                            if (m + 1 < p.M) {
                                if (use_beta) v1 += beta * ccol[m + 1];
                                ccol[m + 1] = v1;
                            }
                        }
                    }
                } else {
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        const int m = m0 + warp_m * 64 + 8 * i + pr;
                        if (m >= p.M) continue;
                        double v = alpha * acc[i][j][jj];
                        if (use_beta) v += beta * ccol[m];
                        ccol[m] = v;
                    }
                }
            }
        }
    }
}

template <bool TA, bool TB>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_f64_dmma_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
                     const Params p) {
    dmma_persistent<TA, TB, false>(mapA, mapB, p, SyrkSched{});
}

// Gramian partials: only the lower-triangle tiles of C = op(A) op(B) with op(B) = op(A)^T, split over K (see SyrkSched).
template <bool TA, bool TB>
__global__ void __launch_bounds__(NUM_THREADS, 1)
syrk_f64_dmma_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
                     const Params p, const SyrkSched sk) {
    dmma_persistent<TA, TB, true>(mapA, mapB, p, sk);
}

// -------------------------------------------------------------------------------------------
// Grouped variant: ONE persistent launch for a rank's whole share of a blocked multiply
// (BlockMatrix.multiply, matrix/BlockMatrix.scala:149-186).  The launch is a list of ENTRIES; an entry is a rectangular
// region of one C block (i,j) — the whole block, a column half, or a (row band x column band) sub-block — with its own
// list of K segments (the kk this rank holds, each an A(i,kk) / B(kk,j) pair), so the reduceByKey over kk (:177)
// happens in the register accumulators and the partial last wave of a per-product launch (an 8192³ product is 4096
// tiles = 31.03 waves on 132 SMs) is paid once per launch, not
// once per product.  All operands are 'N' (column-major blocks).
//
// Three things make the same kernel the compute half of the multi-GPU protocol (csrc/dist.cu):
//   * operand readiness: an operand tile may still be in flight (copy-engine pull over NVLink, or H2D upload) when
//     the kernel starts.  The TMA producer thread polls a per-(tile, band) flag (ld.acquire.gpu) before the first
//     load that touches the band, so the tensor cores start on the bands that have landed;
//   * an entry may add a staged addend: D = acc + Cin, gated by a system-scope flag (the other holder of the C block
//     has finished writing its partial into this GPU's staging buffer), and D may be a PEER pointer: the epilogue's
//     st.global.v2.f64 go over NVLink.  Together: GEMM + reduce-scatter of the k partials in one kernel;
//   * completion: when the last CTA tile of an entry has been stored, one thread publishes a flag (st.release.sys)
//     locally (the D2H stream waits on it) and/or on the peer (its gated entries may start).
// -------------------------------------------------------------------------------------------
struct G2Ent {
    double* D;
    const double* Cin;
    const unsigned long long* cin_flag;
    unsigned long long cin_val;
    unsigned long long* done_ctr;
    unsigned long long* sig_remote;
    unsigned long long* sig_local;
    unsigned long long sig_val;
    long long ldd, ldcin;
    int M, N, m_off, n_off;
    int tiles_m, tiles_n, tile_start, nseg;
    unsigned short nkb[G2_MAX_SEG];
    unsigned char a_op[G2_MAX_SEG], b_op[G2_MAX_SEG];
};

struct G2Params {
    CUtensorMap mapA[G2_MAX_OPS];
    CUtensorMap mapB[G2_MAX_OPS];
    G2Ent e[G2_MAX_ENTRIES];
    int a_band[G2_MAX_OPS], b_band[G2_MAX_OPS];          // rows (A) / columns (B) per readiness band
    short a_ready[G2_MAX_OPS], b_ready[G2_MAX_OPS];      // first flag of the tile in `ready`, or -1 = resident
    const unsigned long long* ready;
    unsigned long long ready_val;
    unsigned long long* status;                           // set to 1 if a wait times out
    long long timeout_ns;
    int ne, num_tiles;
    int poll_mode;                                        // 0: every thread polls the addend flag, 1: lane 0 + __syncwarp
    int fence_all;                                        // 1: every thread fences its stores before the tile is counted
};

__device__ __forceinline__ unsigned long long ld_acquire_gpu(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
// Spin until *flag >= v.  Bounded: after timeout_ns the status word is set and the wait gives up (the result is then
// garbage, the host sees the status word and reports MB_ERR_TIMEOUT instead of hanging the GPU).
template <bool SYS>
__device__ __forceinline__ void wait_flag_ge(const unsigned long long* flag, unsigned long long v, long long timeout_ns,
                                             unsigned long long* status, unsigned long long tag = 1ull) {
    if ((SYS ? ld_acquire_sys(flag) : ld_acquire_gpu(flag)) >= v) return;
    const unsigned long long t0 = globaltimer_ns();
    for (unsigned spins = 0;; ++spins) {
        if ((SYS ? ld_acquire_sys(flag) : ld_acquire_gpu(flag)) >= v) return;
        __nanosleep(64);
        if ((spins & 255u) == 255u && timeout_ns > 0 && (long long)(globaltimer_ns() - t0) > timeout_ns) {
            if (status) *status = tag;
            return;
        }
    }
}

__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_f64_dmma_grouped_kernel(const __grid_constant__ G2Params g) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t bar_full = smem_base + NUM_STAGES * STAGE_BYTES;
    const uint32_t bar_empty = bar_full + NUM_STAGES * 8;
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int num_tiles = g.num_tiles;

    if (threadIdx.x == 0) {
        for (int s = 0; s < NUM_STAGES; ++s) {
            mbar_init(bar_full + 8 * s, 1);
            mbar_init(bar_empty + 8 * s, NUM_CONSUMER_WARPS);
        }
        fence_barrier_init();
    }
    __syncthreads();

    auto locate = [&](int t, int& c, int& tm, int& tn) {
        c = 0;
        while (c + 1 < g.ne && t >= g.e[c + 1].tile_start) ++c;
        tile_coords(t - g.e[c].tile_start, g.e[c].tiles_m, g.e[c].tiles_n, tm, tn);
    };

    if (warp < 4) {
        setmaxnreg_dec<40>();
        if (warp == 0 && lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
                int c, tm, tn;
                locate(t, c, tm, tn);
                const G2Ent& en = g.e[c];
                const int m0 = en.m_off + tm * BM, n0 = en.n_off + tn * BN;
                for (int sg = 0; sg < en.nseg; ++sg) {
                    const int ia = en.a_op[sg], ib = en.b_op[sg];
                    // operand bands still in flight?  (pulled / uploaded tiles only; resident tiles have ready = -1)
                    if (g.a_ready[ia] >= 0)
                        wait_flag_ge<false>(g.ready + g.a_ready[ia] + m0 / g.a_band[ia], g.ready_val, g.timeout_ns, g.status,
                                            (1ull << 56) | (1ull << 48) | (unsigned long long)(g.a_ready[ia] + m0 / g.a_band[ia]));
                    if (g.b_ready[ib] >= 0)
                        wait_flag_ge<false>(g.ready + g.b_ready[ib] + n0 / g.b_band[ib], g.ready_val, g.timeout_ns, g.status,
                                            (1ull << 56) | (2ull << 48) | (unsigned long long)(g.b_ready[ib] + n0 / g.b_band[ib]));
                    const CUtensorMap* mA = &g.mapA[ia];
                    const CUtensorMap* mB = &g.mapB[ib];
                    const int nkb = en.nkb[sg];
                    for (int kb = 0; kb < nkb; ++kb) {
                        mbar_wait(bar_empty + 8 * stage, phase ^ 1);
                        const uint32_t full = bar_full + 8 * stage;
                        const uint32_t sA = smem_base + stage * STAGE_BYTES;
                        const uint32_t sB = sA + OPERAND_BYTES;
                        mbar_arrive_expect_tx(full, STAGE_BYTES);
                        const int k0 = kb * BK;
#pragma unroll
                        for (int b = 0; b < 8; ++b) tma_load_2d(sA + b * 2048, mA, full, m0 + 16 * b, k0);
                        tma_load_2d(sB, mB, full, k0, n0);
                        if (++stage == NUM_STAGES) { stage = 0; phase ^= 1; }
                    }
                }
            }
        }
        return;
    }

    setmaxnreg_inc<232>();
    const int cw = warp - 4;
    const int warp_m = cw & 1;
    const int warp_n = cw >> 1;
    const int r = lane >> 2;
    const int q = lane & 3;
    const int pr = perm8(r);
    uint32_t offA[2][2], offB[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int pp = 0; pp < 2; ++pp) {
            const int krow = 8 * h + 2 * q + pp;
            offA[h][pp] = warp_m * 4 * 2048 + krow * 128 + ((r ^ (krow & 7)) << 4);
        }
        offB[h] = warp_n * 32 * 128 + pr * 128 + ((((4 * h + q) ^ pr) & 7) << 4);
    }

    int stage = 0;
    uint32_t phase = 0;
    const unsigned long long* cin_seen = nullptr;      // last addend flag this thread has already observed
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        int c, tm_, tn_;
        locate(t, c, tm_, tn_);
        const G2Ent& en = g.e[c];
        const int m0 = tm_ * BM, n0 = tn_ * BN;       // relative to the entry's region
        int total_kb = 0;
        for (int sg = 0; sg < en.nseg; ++sg) total_kb += en.nkb[sg];
        double acc[8][4][2];
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;

        for (int kb = 0; kb < total_kb; ++kb) {
            mbar_wait(bar_full + 8 * stage, phase);
            const uint32_t sA = smem_base + stage * STAGE_BYTES;
            const uint32_t sB = sA + OPERAND_BYTES;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                double a[8][2], b[4][2];
#pragma unroll
                for (int tp = 0; tp < 4; ++tp)
#pragma unroll
                    for (int pp = 0; pp < 2; ++pp) lds128(a[2 * tp][pp], a[2 * tp + 1][pp], sA + offA[h][pp] + tp * 2048);
#pragma unroll
                for (int u = 0; u < 4; ++u) lds128(b[u][0], b[u][1], sB + offB[h] + u * 8 * 128);
                if (h == 1) {
                    __syncwarp();
                    if (lane == 0) mbar_arrive(bar_empty + 8 * stage);
                }
#pragma unroll
                for (int pp = 0; pp < 2; ++pp)
#pragma unroll
                    for (int i = 0; i < 8; ++i)
#pragma unroll
                        for (int j = 0; j < 4; ++j) dmma_m8n8k4(acc[i][j][0], acc[i][j][1], a[i][pp], b[j][pp]);
            }
            if (++stage == NUM_STAGES) { stage = 0; phase ^= 1; }
        }

        // ---------------- epilogue: D = acc (+ Cin) ----------------
        double* Db = en.D;
        const double* Ci = en.Cin;
        const long long ldd = en.ldd, ldci = en.ldcin;
        const int Mc = en.M, Nc = en.N;
        if (Ci != nullptr && en.cin_flag != nullptr && en.cin_flag != cin_seen) {
            // the other holder's partial must have landed in this GPU's staging buffer (every lane acquires)
            if (g.poll_mode == 0 || lane == 0)
                wait_flag_ge<true>(en.cin_flag, en.cin_val, g.timeout_ns, g.status, (1ull << 56) | (3ull << 48) | (unsigned long long)c);
            if (g.poll_mode != 0) __syncwarp();
            cin_seen = en.cin_flag;
        }
        const bool vec_ok = ((reinterpret_cast<uintptr_t>(Db) & 15) == 0) && ((ldd & 1) == 0) &&
                            (Ci == nullptr || (((reinterpret_cast<uintptr_t>(Ci) & 15) == 0) && ((ldci & 1) == 0)));
#pragma unroll
        for (int j = 0; j < 4; ++j) {
#pragma unroll
            for (int jj = 0; jj < 2; ++jj) {
                const int n = n0 + warp_n * 32 + 8 * j + perm8(2 * q + jj);
                if (n >= Nc) continue;
                double* dcol = Db + (long long)n * ldd;
                const double* ccol = Ci ? Ci + (long long)n * ldci : nullptr;
#pragma unroll
                for (int tp = 0; tp < 4; ++tp) {
                    const int m = m0 + warp_m * 64 + 16 * tp + 2 * r;
                    if (m >= Mc) continue;
                    double v0 = acc[2 * tp][j][jj], v1 = acc[2 * tp + 1][j][jj];
                    if (vec_ok && m + 1 < Mc) {
                        if (ccol) {
                            const double2 old = __ldcg(reinterpret_cast<const double2*>(ccol + m));
                            v0 += old.x;
                            v1 += old.y;
                        }
                        *reinterpret_cast<double2*>(dcol + m) = make_double2(v0, v1);
                    } else {
                        if (ccol) v0 += __ldcg(ccol + m);
                        dcol[m] = v0;
                        if (m + 1 < Mc) {
                            if (ccol) v1 += __ldcg(ccol + m + 1);
                            dcol[m + 1] = v1;
                        }
                    }
                }
            }
        }
        if (en.done_ctr != nullptr) {
            // every consumer thread's stores of this tile, then ONE thread counts the tile and, if it was the entry's last,
            // publishes the completion flags with system scope (peer GPUs and the copy streams poll them).
            // EVERY thread fences its own stores first (the conservative order: fence, CTA barrier, count).  NOTE: with the
            // tile stored to a PEER GPU this sequence was still measured faulty — one 16x32 patch of a tile stale in about a
            // third of the 8192^2 calls, with or without the per-thread fences — so csrc/dist.cu only arms done_ctr for entries whose output is in
            // LOCAL memory; peer outputs are announced by a stream memory operation after the launch (two-launch
            // reduce-scatter) or pushed by the copy engine (host path).  The single-launch form stays behind
            // MARLIN_B200_FUSED_SPLIT=0 for the investigation.
            if (g.fence_all) __threadfence_system();
            asm volatile("bar.sync 1, %0;" ::"n"(NUM_CONSUMER_WARPS * 32) : "memory");
            if (cw == 0 && lane == 0) {
                __threadfence_system();
                const unsigned long long prev = atomicAdd(en.done_ctr, 1ull);
                if (prev + 1ull == (unsigned long long)(en.tiles_m * en.tiles_n)) {
                    __threadfence_system();
                    if (en.sig_remote) asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(en.sig_remote), "l"(en.sig_val) : "memory");
                    if (en.sig_local) asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(en.sig_local), "l"(en.sig_val) : "memory");
                }
            }
        }
    }
}

// -------------------------------------------------------------------------------------------
// Generic CUDA-core kernel: any ld / offset / alignment, any trans.  64x64 tile, 4x4 per thread.
// Used when TMA's 16-byte rules do not hold (odd leading dimension or odd element offset of a
// Breeze view) and as an independent on-device cross-check in the tests.
// -------------------------------------------------------------------------------------------
template <bool TA, bool TB>
__global__ void __launch_bounds__(256)
gemm_f64_generic_kernel(int M, int N, int K, double alpha, const double* __restrict__ A, long long lda,
                        const double* __restrict__ B, long long ldb, double beta, double* __restrict__ C,
                        long long ldc) {
    constexpr int T = 64, KK = 16;
    __shared__ double sA[KK][T + 1];
    __shared__ double sB[KK][T + 1];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int m0 = blockIdx.x * T, n0 = blockIdx.y * T;
    double acc[4][4] = {};
    for (int k0 = 0; k0 < K; k0 += KK) {
        for (int e = threadIdx.x; e < T * KK; e += 256) {
            // A tile element (m, k)
            int mm, kk;
            if (!TA) { mm = e % T; kk = e / T; } else { kk = e % KK; mm = e / KK; }
            const int gm = m0 + mm, gk = k0 + kk;
            double v = 0.0;
            if (gm < M && gk < K) v = !TA ? A[gm + (long long)gk * lda] : A[gk + (long long)gm * lda];
            sA[kk][mm] = v;
            int nn, kb;
            if (!TB) { kb = e % KK; nn = e / KK; } else { nn = e % T; kb = e / T; }
            const int gn = n0 + nn, gk2 = k0 + kb;
            double w = 0.0;
            if (gn < N && gk2 < K) w = !TB ? B[gk2 + (long long)gn * ldb] : B[gn + (long long)gk2 * ldb];
            sB[kb][nn] = w;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < KK; ++kk) {
            double a[4], b[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = sA[kk][tx + 16 * i];
#pragma unroll
            for (int j = 0; j < 4; ++j) b[j] = sB[kk][ty + 16 * j];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fma(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int n = n0 + ty + 16 * j;
        if (n >= N) continue;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int m = m0 + tx + 16 * i;
            if (m >= M) continue;
            double v = alpha * acc[i][j];
            double* c = C + m + (long long)n * ldc;
            if (beta != 0.0) v += beta * *c;
            *c = v;
        }
    }
}

__global__ void scale_matrix_kernel(int M, int N, double beta, double* C, long long ldc) {
    const long long total = (long long)M * N;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total;
         e += (long long)gridDim.x * blockDim.x) {
        const long long m = e % M, n = e / M;
        double* c = C + m + n * ldc;
        *c = (beta == 0.0) ? 0.0 : beta * *c;
    }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(ptr);
    }
    return fn;
}

// 2-D fp64 tensor map over a column-major array: dim0 (contiguous) x dim1 (stride ld), 128B swizzle.
bool make_map_f64(CUtensorMap* map, const double* base, uint64_t dim0, uint64_t dim1, uint64_t ld,
                  uint32_t box0, uint32_t box1) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) return false;
    cuuint64_t dims[2] = {dim0, dim1};
    cuuint64_t strides[1] = {ld * 8};
    cuuint32_t box[2] = {box0, box1};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 2, const_cast<double*>(base), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

template <bool TA, bool TB>
cudaError_t launch_dmma(const CUtensorMap& mA, const CUtensorMap& mB, const Params& p, int num_sms,
                        cudaStream_t stream) {
    auto kern = gemm_f64_dmma_kernel<TA, TB>;
    // per template instantiation; idempotent, so concurrent first calls may both set it (no unsynchronised flag)
    static std::atomic<bool> attr_done{false};
    if (!attr_done.load(std::memory_order_acquire)) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
        if (e != cudaSuccess) return e;
        attr_done.store(true, std::memory_order_release);
    }
    const int grid = min(p.tiles_m * p.tiles_n, num_sms);
    kern<<<grid, NUM_THREADS, SMEM_BYTES, stream>>>(mA, mB, p);
    return cudaGetLastError();
}

}  // namespace

bool gemm_f64_tma_eligible(const double* A, long long lda, const double* B, long long ldb) {
    return ((reinterpret_cast<uintptr_t>(A) & 15) == 0) && ((reinterpret_cast<uintptr_t>(B) & 15) == 0) &&
           (lda % 2 == 0) && (ldb % 2 == 0) && get_encode_fn() != nullptr;
}

cudaError_t gemm_f64(bool transA, bool transB, int M, int N, int K, double alpha, const double* A, long long lda,
                     const double* B, long long ldb, double beta, double* C, long long ldc, int num_sms,
                     cudaStream_t stream, bool force_generic, int* launches) {
    if (M <= 0 || N <= 0) return cudaSuccess;
    if (K <= 0 || alpha == 0.0) {
        if (beta == 1.0) return cudaSuccess;
        scale_matrix_kernel<<<min(1184, (int)(((long long)M * N + 255) / 256)), 256, 0, stream>>>(M, N, beta, C, ldc);
        if (launches) ++*launches;
        return cudaGetLastError();
    }
    if (!force_generic && gemm_f64_tma_eligible(A, lda, B, ldb)) {
        CUtensorMap mA, mB;
        bool ok = true;
        // A: 'N' -> stored M x K (m contiguous), MN form boxes [16 m][16 k]; 'T' -> stored K x M, K form box [16 k][128 m]
        ok = ok && (!transA ? make_map_f64(&mA, A, M, K, lda, 16, 16) : make_map_f64(&mA, A, K, M, lda, 16, 128));
        // B: 'N' -> stored K x N (k contiguous), K form box [16 k][128 n]; 'T' -> stored N x K, MN form boxes [16 n][16 k]
        ok = ok && (!transB ? make_map_f64(&mB, B, K, N, ldb, 16, 128) : make_map_f64(&mB, B, N, K, ldb, 16, 16));
        if (ok) {
            Params p;
            p.M = M; p.N = N; p.K = K; p.alpha = alpha; p.beta = beta; p.C = C; p.ldc = ldc;
            p.tiles_m = (M + BM - 1) / BM;
            p.tiles_n = (N + BN - 1) / BN;
            if (launches) ++*launches;
            if (!transA && !transB) return launch_dmma<false, false>(mA, mB, p, num_sms, stream);
            if (transA && !transB) return launch_dmma<true, false>(mA, mB, p, num_sms, stream);
            if (!transA && transB) return launch_dmma<false, true>(mA, mB, p, num_sms, stream);
            return launch_dmma<true, true>(mA, mB, p, num_sms, stream);
        }
    }
    dim3 grid((M + 63) / 64, (N + 63) / 64);
    if (launches) ++*launches;
    if (!transA && !transB)
        gemm_f64_generic_kernel<false, false><<<grid, 256, 0, stream>>>(M, N, K, alpha, A, lda, B, ldb, beta, C, ldc);
    else if (transA && !transB)
        gemm_f64_generic_kernel<true, false><<<grid, 256, 0, stream>>>(M, N, K, alpha, A, lda, B, ldb, beta, C, ldc);
    else if (!transA && transB)
        gemm_f64_generic_kernel<false, true><<<grid, 256, 0, stream>>>(M, N, K, alpha, A, lda, B, ldb, beta, C, ldc);
    else
        gemm_f64_generic_kernel<true, true><<<grid, 256, 0, stream>>>(M, N, K, alpha, A, lda, B, ldb, beta, C, ldc);
    return cudaGetLastError();
}


// ---------------------------------------------------------------------------------------------------------------------
// Gramian G = op(A) op(A)^T (DenseVecMatrix.computeGramianMatrix, matrix/DenseVecMatrix.scala:1464-1486).
// ---------------------------------------------------------------------------------------------------------------------
namespace {

// Sum the split-K partials of lower 32x32 tile (bi, bj), bi >= bj, in split order and store it to G(bi, bj) and, through a
// shared-memory transpose, to G(bj, bi): G is exactly symmetric and does not depend on the launch order of the partials.
// With one split the "partial" may be G itself (ws == G, ldw == ldg): a CTA reads only its own lower tile (and, on the
// diagonal, its own whole tile) before its barrier and no other CTA reads what it writes, so the pass runs in place.
// Accesses are 128-bit where alignment and the leading dimensions allow.
template <bool VEC_W>
__global__ void __launch_bounds__(256) gram_reduce_mirror_kernel(const double* ws, long long ldw, long long stride,
                                                                 int splits, int n, double* G, long long ldg) {
    __shared__ double tile[32][33];          // [column][row] of the summed lower tile
    int bi, bj;
    tri_coords(blockIdx.x, bi, bj);
    const int r0 = bi * 32, c0 = bj * 32;
    const int rp = threadIdx.x & 15, cy = threadIdx.x >> 4;
    const bool vec_g = ((reinterpret_cast<uintptr_t>(G) & 15) == 0) && ((ldg & 1) == 0);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int c = cy + 16 * i, r = 2 * rp;
        double2 acc = make_double2(0.0, 0.0);
        if (c0 + c < n && r0 + r < n) {
            const double* src = ws + (r0 + r) + (long long)(c0 + c) * ldw;
            const bool second = r0 + r + 1 < n;
            for (int s = 0; s < splits; ++s) {
                if (VEC_W) {
                    const double2 v = *reinterpret_cast<const double2*>(src + s * stride);
                    acc.x += v.x;
                    acc.y += v.y;
                } else {
                    acc.x += src[s * stride];
                    if (second) acc.y += src[s * stride + 1];
                }
            }
        }
        tile[c][r] = acc.x;
        tile[c][r + 1] = acc.y;
    }
    __syncthreads();
    auto store2 = [&](int row, int col, double v0, double v1, bool w0, bool w1) {
        double* dst = G + row + (long long)col * ldg;
        if (w0 && w1 && vec_g) {
            *reinterpret_cast<double2*>(dst) = make_double2(v0, v1);
        } else {
            if (w0) dst[0] = v0;
            if (w1) dst[1] = v1;
        }
    };
    const bool diag = bi == bj;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int y = cy + 16 * i, x = 2 * rp;
        // direct: G(r0 + x + e, c0 + y), the lower part (row >= col) of a diagonal tile
        if (c0 + y < n) {
            const bool w0 = r0 + x < n && (!diag || x >= y), w1 = r0 + x + 1 < n && (!diag || x + 1 >= y);
            store2(r0 + x, c0 + y, tile[y][x], tile[y][x + 1], w0, w1);
        }
        // mirrored: G(c0 + x + e, r0 + y) = S(r0 + y, c0 + x + e), the strict upper part of a diagonal tile
        if (r0 + y < n) {
            const bool w0 = c0 + x < n && (!diag || x < y), w1 = c0 + x + 1 < n && (!diag || x + 1 < y);
            store2(c0 + x, r0 + y, tile[x][y], tile[x + 1][y], w0, w1);
        }
    }
}

}  // namespace

// Split K only when the lower triangle has too few tiles to keep the SMs busy (fewer than two waves), and only as far as
// the partials fit in GRAM_WS_CAP_DOUBLES: the smallest split that fills the last wave best, a larger one only for at
// least 1 % more fill, and >= 512 rows per split.  Above 22 tile rows (n > 2816 on 132 SMs) this is always 1 split and
// the Gramian needs no workspace at all.
int gram_splits(int n, long long K, int num_sms) {
    if (n <= 0 || num_sms <= 0) return 1;
    const long long t = (n + BM - 1) / BM;
    const long long tri = t * (t + 1) / 2;
    if (tri >= 2LL * num_sms) return 1;
    const long long ldw = (n + 1) & ~1;
    const long long kb = (K + BK - 1) / BK;
    const long long cap = std::min<long long>(32, GRAM_WS_CAP_DOUBLES / (ldw * n));
    int best = 1;
    double best_eff = (double)tri / (double)(((tri + num_sms - 1) / num_sms) * num_sms);
    for (int s = 2; s <= cap; ++s) {
        if (kb / s < 32) break;                               // keep >= 512 rows per split
        const long long items = tri * s;
        const long long waves = (items + num_sms - 1) / num_sms;
        const double eff = (double)items / (double)(waves * num_sms);
        if (eff >= best_eff + 0.01) { best_eff = eff; best = s; }
    }
    return best;
}

size_t gram_workspace_doubles(int n, long long K, int num_sms) {
    const int s = gram_splits(n, K, num_sms);
    return s > 1 ? (size_t)s * (size_t)((n + 1) & ~1) * (size_t)n : 0;
}

cudaError_t gram_f64(bool trans, int n, int K, const double* A, long long lda, double* G, long long ldg, double* ws,
                     int num_sms, cudaStream_t stream, int* launches) {
    if (n <= 0) return cudaSuccess;
    CUtensorMap mA, mB;
    const bool tma = K > 0 && gemm_f64_tma_eligible(A, lda, A, lda) &&
                     (!trans ? (make_map_f64(&mA, A, n, K, lda, 16, 16) && make_map_f64(&mB, A, n, K, lda, 16, 16))
                             : (make_map_f64(&mA, A, K, n, lda, 16, 128) && make_map_f64(&mB, A, K, n, lda, 16, 128)));
    const int splits = tma ? gram_splits(n, K, num_sms) : 1;
    if (splits > 1 && ws == nullptr) return cudaErrorInvalidValue;
    // one split: the product goes straight into G and the mirror pass runs in place
    double* P = splits > 1 ? ws : G;
    const long long ldp = splits > 1 ? ((n + 1) & ~1) : ldg;
    cudaError_t e;
    if (tma) {
        const int t = (n + BM - 1) / BM;
        const long long kb = (K + BK - 1) / BK;
        Params p;
        p.M = n; p.N = n; p.K = K; p.alpha = 1.0; p.beta = 0.0; p.C = P; p.ldc = ldp;
        p.tiles_m = t; p.tiles_n = t;
        SyrkSched sk;
        sk.splits = splits;
        sk.tri_tiles = t * (t + 1) / 2;
        sk.kchunk = (int)((kb + splits - 1) / splits) * BK;
        sk.split_stride = ldp * n;
        auto kern = !trans ? syrk_f64_dmma_kernel<false, true> : syrk_f64_dmma_kernel<true, false>;
        e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
        if (e != cudaSuccess) return e;
        kern<<<min(sk.tri_tiles * splits, num_sms), NUM_THREADS, SMEM_BYTES, stream>>>(mA, mB, p, sk);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
        if (launches) ++*launches;
    } else {
        // the whole product on the CUDA cores (views TMA cannot address), or zeros for K = 0
        e = gemm_f64(trans, !trans, n, n, K, 1.0, A, lda, A, lda, 0.0, P, ldp, num_sms, stream, true, launches);
        if (e != cudaSuccess) return e;
    }
    const int nb = (n + 31) / 32;
    const unsigned grid = nb * (nb + 1) / 2;
    if (((reinterpret_cast<uintptr_t>(P) & 15) == 0) && ((ldp & 1) == 0))
        gram_reduce_mirror_kernel<true><<<grid, 256, 0, stream>>>(P, ldp, ldp * n, splits, n, G, ldg);
    else
        gram_reduce_mirror_kernel<false><<<grid, 256, 0, stream>>>(P, ldp, ldp * n, splits, n, G, ldg);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t gemm_f64_grouped2(const G2Launch& L, int num_sms, cudaStream_t stream, int* launches) {
    if (L.ne <= 0) return cudaSuccess;
    if (L.ne > G2_MAX_ENTRIES || L.na > G2_MAX_OPS || L.nb > G2_MAX_OPS || !get_encode_fn()) return cudaErrorNotSupported;
    static thread_local G2Params g;          // ~20 KB parameter block: kept off the stack, one per calling thread
    for (int i = 0; i < L.na; ++i) {
        const G2Operand& o = L.A[i];
        if (o.rows <= 0 || o.cols <= 0 || !gemm_f64_tma_eligible(o.ptr, o.ld, o.ptr, 2)) return cudaErrorNotSupported;
        if (!make_map_f64(&g.mapA[i], o.ptr, o.rows, o.cols, o.ld, 16, 16)) return cudaErrorNotSupported;
        if (o.ready_base >= 0 && (o.band <= 0 || o.band % BM != 0)) return cudaErrorInvalidValue;
        g.a_band[i] = o.band > 0 ? o.band : (1 << 30);
        g.a_ready[i] = (short)o.ready_base;
    }
    for (int i = 0; i < L.nb; ++i) {
        const G2Operand& o = L.B[i];
        if (o.rows <= 0 || o.cols <= 0 || !gemm_f64_tma_eligible(o.ptr, o.ld, o.ptr, 2)) return cudaErrorNotSupported;
        if (!make_map_f64(&g.mapB[i], o.ptr, o.rows, o.cols, o.ld, 16, 128)) return cudaErrorNotSupported;
        if (o.ready_base >= 0 && (o.band <= 0 || o.band % BN != 0)) return cudaErrorInvalidValue;
        g.b_band[i] = o.band > 0 ? o.band : (1 << 30);
        g.b_ready[i] = (short)o.ready_base;
    }
    int tiles = 0;
    for (int c = 0; c < L.ne; ++c) {
        const G2Entry& s = L.E[c];
        G2Ent& d = g.e[c];
        if (s.nseg <= 0 || s.nseg > G2_MAX_SEG || s.M <= 0 || s.N <= 0) return cudaErrorNotSupported;
        if ((s.m_off % BM) != 0 || (s.n_off % BN) != 0) return cudaErrorInvalidValue;
        d.D = s.D; d.ldd = s.ldd; d.Cin = s.Cin; d.ldcin = s.ldcin;
        d.cin_flag = s.cin_flag; d.cin_val = s.cin_val;
        d.done_ctr = s.done_ctr; d.sig_remote = s.sig_remote; d.sig_local = s.sig_local; d.sig_val = s.sig_val;
        d.M = s.M; d.N = s.N; d.m_off = s.m_off; d.n_off = s.n_off;
        d.tiles_m = (s.M + BM - 1) / BM;
        d.tiles_n = (s.N + BN - 1) / BN;
        d.tile_start = tiles;
        tiles += d.tiles_m * d.tiles_n;
        d.nseg = s.nseg;
        for (int sg = 0; sg < s.nseg; ++sg) {
            const int ia = s.a_op[sg], ib = s.b_op[sg];
            if (ia < 0 || ia >= L.na || ib < 0 || ib >= L.nb || L.A[ia].cols != L.B[ib].rows) return cudaErrorInvalidValue;
            const int nkb = (L.A[ia].cols + BK - 1) / BK;
            if (nkb > 65535) return cudaErrorNotSupported;
            d.nkb[sg] = (unsigned short)nkb;
            d.a_op[sg] = (unsigned char)ia;
            d.b_op[sg] = (unsigned char)ib;
        }
    }
    g.ready = L.ready; g.ready_val = L.ready_val; g.status = L.status; g.timeout_ns = L.timeout_ns;
    g.ne = L.ne;
    g.num_tiles = tiles;
    static const int fence_all = [] { const char* e = getenv("MARLIN_B200_FENCE_ALL"); return (e && e[0] == '0') ? 0 : 1; }();
    g.fence_all = fence_all;
    static const int poll_mode = [] { const char* e = getenv("MARLIN_B200_CIN_POLL"); return (e && e[0] == '1') ? 1 : 0; }();
    g.poll_mode = poll_mode;
    static std::atomic<bool> attr_done{false};
    if (!attr_done.load(std::memory_order_acquire)) {
        cudaError_t e = cudaFuncSetAttribute(gemm_f64_dmma_grouped_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
        if (e != cudaSuccess) return e;
        attr_done.store(true, std::memory_order_release);
    }
    const int grid = min(tiles, num_sms);
    gemm_f64_dmma_grouped_kernel<<<grid, NUM_THREADS, SMEM_BYTES, stream>>>(g);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t gemm_f64_grouped(int m, int k, int n, const int* my_c, int num_c, const double* const* A, const long long* lda,
                             const double* const* B, const long long* ldb, double* const* C, const long long* ldc,
                             const int* row_len, const int* k_len, const int* col_len, int num_sms, cudaStream_t stream,
                             int* launches) {
    // my_c: the (i*n + j) ids of the C blocks to compute; A[i*k+kk], B[kk*n+j], C[i*n+j] column-major 'N' blocks.
    // One entry per C block (the whole block, every kk), operands resident: no flags, no addend.
    if (num_c <= 0) return cudaSuccess;
    if (num_c > G2_MAX_ENTRIES || k > G2_MAX_SEG) return cudaErrorNotSupported;
    static thread_local G2Launch L;
    L = G2Launch();
    int a_of_row[G2_MAX_ENTRIES], b_of_col[G2_MAX_ENTRIES], rows_seen[G2_MAX_ENTRIES], cols_seen[G2_MAX_ENTRIES], nrows = 0, ncols = 0;
    for (int c = 0; c < num_c; ++c) {
        const int i = my_c[c] / n, j = my_c[c] % n;
        if (row_len[i] <= 0 || col_len[j] <= 0) return cudaErrorNotSupported;
        int ri = -1, cj = -1;
        for (int x = 0; x < nrows; ++x) if (rows_seen[x] == i) ri = x;
        for (int x = 0; x < ncols; ++x) if (cols_seen[x] == j) cj = x;
        if (ri < 0) {
            if (L.na + k > G2_MAX_OPS) return cudaErrorNotSupported;
            for (int kk = 0; kk < k; ++kk) {
                if (k_len[kk] <= 0) return cudaErrorNotSupported;
                G2Operand& o = L.A[L.na + kk];
                o.ptr = A[i * k + kk]; o.ld = lda[i * k + kk]; o.rows = row_len[i]; o.cols = k_len[kk]; o.band = 0; o.ready_base = -1;
            }
            rows_seen[nrows] = i; a_of_row[nrows] = L.na; ri = nrows++; L.na += k;
        }
        if (cj < 0) {
            if (L.nb + k > G2_MAX_OPS) return cudaErrorNotSupported;
            for (int kk = 0; kk < k; ++kk) {
                G2Operand& o = L.B[L.nb + kk];
                o.ptr = B[kk * n + j]; o.ld = ldb[kk * n + j]; o.rows = k_len[kk]; o.cols = col_len[j]; o.band = 0; o.ready_base = -1;
            }
            cols_seen[ncols] = j; b_of_col[ncols] = L.nb; cj = ncols++; L.nb += k;
        }
        G2Entry& e = L.E[L.ne++];
        e.nseg = k;
        for (int kk = 0; kk < k; ++kk) { e.a_op[kk] = a_of_row[ri] + kk; e.b_op[kk] = b_of_col[cj] + kk; }
        e.M = row_len[i]; e.N = col_len[j];
        e.D = C[my_c[c]]; e.ldd = ldc[my_c[c]];
    }
    return gemm_f64_grouped2(L, num_sms, stream, launches);
}

}  // namespace mb

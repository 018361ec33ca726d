// fp64 block GEMM for sm_90a — replaces SubMatrix.multiply -> Breeze `*` -> netlib dgemm
// (reference: matrix/SubMatrix.scala:87-91; inline twins matrix/DenseVecMatrix.scala:122,129,1676).
//
// wgmma has no fp64 type, so the fp64 tensor-core path on H100 is DMMA: mma.sync.m16n8k4.f64 (SASS DMMA.16x8x4), which
// issues at twice the rate of the Ampere shape m8n8k4 (SASS DMMA.8x8x4).  Design:
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
// contiguous dimension is K ("K form") as one box of [128 mn-rows][16 k] (operand_map).
//
// Three kernels run this mainloop: gemm_f64_dmma16x8_kernel (every tile of C), syrk_f64_dmma16x8_kernel (the Gramian's
// lower-triangle tiles, split over K) and gemm_f64_dmma16x8_grouped_kernel (a list of C regions, each over its own K
// segments).  They share one set of pieces, templated on the operands' forms: ring_setup, load_slab (producer),
// consumer_lane + mma_slab (consumers) and store_tile (epilogue).  Each kernel keeps only its tile schedule, its K
// range and what its epilogue waits for or signals.
//
// Each of the three also exists as an m8n8k4 instance under its older name (gemm_f64_dmma_kernel, syrk_f64_dmma_kernel,
// gemm_f64_dmma_grouped_kernel): the same source with only the instruction shape changed (mma_slab).  m16n8k4 is two
// m8n8k4 stacked in M that share the B fragment, so both shapes give every element of C the same 4-term steps over the
// same k in the same order, and the results are identical bit for bit.  The m8n8k4 instances are the in-library
// reference of the production kernels and run only when a context asks for them (mb_set_dmma_reference).
#include "gemm_f64.h"
#include "ptx.cuh"
#include "launch.h"
#include "tma.h"
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

// The DMMA instruction shape of the mainloop: m16n8k4 in production, m8n8k4 for the reference instances.
enum class Dmma { m8n8k4, m16n8k4 };

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

// ---- the mainloop pieces of the three DMMA kernels.  A is in MN form when !TA, B when TB. ----

// NUM_STAGES stages of [A tile | B tile] from a 1024-byte aligned base (SWIZZLE_128B needs it), then the full and the
// empty mbarrier of every stage.
struct Ring {
    uint32_t base, full, empty;
};

// Thread 0 initialises the barriers and prefetches the descriptors it is given; every thread returns after the CTA barrier.
__device__ __forceinline__ Ring ring_setup(const CUtensorMap* prefetchA, const CUtensorMap* prefetchB) {
    extern __shared__ uint8_t smem_raw[];
    Ring ring;
    ring.base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    ring.full = ring.base + NUM_STAGES * STAGE_BYTES;
    ring.empty = ring.full + NUM_STAGES * 8;
    if (threadIdx.x == 0) {
        for (int s = 0; s < NUM_STAGES; ++s) {
            mbar_init(ring.full + 8 * s, 1);
            mbar_init(ring.empty + 8 * s, NUM_CONSUMER_WARPS);
        }
        fence_barrier_init();
        if (prefetchA) tma_prefetch_desc(prefetchA);
        if (prefetchB) tma_prefetch_desc(prefetchB);
    }
    __syncthreads();
    return ring;
}

// Producer: wait until `stage` is free (its empty barrier completed the phase of parity empty_parity, the producer's
// own phase ^ 1), then load k16 slab kb of the A tile at row m0 and of the B tile at column n0 into it.
template <bool TA, bool TB>
__device__ __forceinline__ void load_slab(const Ring& ring, int stage, uint32_t empty_parity, const CUtensorMap* mapA,
                                          const CUtensorMap* mapB, int m0, int n0, int kb) {
    mbar_wait(ring.empty + 8 * stage, empty_parity);
    const uint32_t full = ring.full + 8 * stage;
    const uint32_t sA = ring.base + stage * STAGE_BYTES;
    const uint32_t sB = sA + OPERAND_BYTES;
    mbar_arrive_expect_tx(full, STAGE_BYTES);
    const int k0 = kb * BK;
    if (!TA) {
#pragma unroll
        for (int b = 0; b < 8; ++b) tma_load_2d(sA + b * 2048, mapA, full, m0 + 16 * b, k0);
    } else {
        tma_load_2d(sA, mapA, full, k0, m0);
    }
    if (!TB) {
        tma_load_2d(sB, mapB, full, k0, n0);
    } else {
#pragma unroll
        for (int b = 0; b < 8; ++b) tma_load_2d(sB + b * 2048, mapB, full, n0 + 16 * b, k0);
    }
}

// A consumer thread: its 64x32 warp tile (warp_m: 64-row slab, warp_n: 32-column slab), its MMA row (A) / column (B) r
// and k slot q, and the byte offsets of its fragment loads inside one operand tile, [h][p] for an MN-form operand and
// [h][0] for a K-form one:
//  MN form: box t' (16 mn x 16 k, 2 KiB), k-row = 8h + 2q + p, 16B chunk = r ^ ((2q+p)&7)
//           -> doubles (mn = 16t' + 2r, 16t' + 2r + 1)  = MMA tiles 2t', 2t'+1, row r.
//  K  form: row mn = base + 8u + perm8(r), 16B chunk = (4h + q) ^ perm8(r)
//           -> doubles (k = 8h + 2q, 8h + 2q + 1)       = phases p = 0, 1.
struct Consumer {
    int lane, warp_m, warp_n, r, q;
    uint32_t offA[2][2], offB[2][2];
};

template <bool TA, bool TB>
__device__ __forceinline__ Consumer consumer_lane(int cw, int lane) {
    Consumer c;
    c.lane = lane;
    c.warp_m = cw & 1;
    c.warp_n = cw >> 1;
    c.r = lane >> 2;
    c.q = lane & 3;
    const int pr = perm8(c.r);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int pp = 0; pp < 2; ++pp) {
            const int krow = 8 * h + 2 * c.q + pp;
            const uint32_t mn_off = krow * 128 + ((c.r ^ (krow & 7)) << 4);
            const uint32_t k_off = pr * 128 + ((((4 * h + c.q) ^ pr) & 7) << 4);
            c.offA[h][pp] = !TA ? (c.warp_m * 4 * 2048 + mn_off) : (c.warp_m * 64 * 128 + k_off);
            c.offB[h][pp] = TB ? (c.warp_n * 2 * 2048 + mn_off) : (c.warp_n * 32 * 128 + k_off);
        }
    }
    return c;
}

// Consumer: wait for the slab in `stage`, read the fragments (24 LDS.128 per warp), hand the stage back to the producer
// and issue the slab into acc: 128 m8n8k4, or 64 m16n8k4 that each take m-tiles 2i' and 2i'+1 together (for an MN-form
// A the two a values come from one LDS.128 and are adjacent registers already).
template <Dmma S, bool TA, bool TB>
__device__ __forceinline__ void mma_slab(double (&acc)[8][4][2], const Ring& ring, int stage, uint32_t phase,
                                         const Consumer c) {
    mbar_wait(ring.full + 8 * stage, phase);
    const uint32_t sA = ring.base + stage * STAGE_BYTES;
    const uint32_t sB = sA + OPERAND_BYTES;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        double a[8][2];   // [m-tile][phase]
        double b[4][2];   // [n-tile][phase]
        if (!TA) {
#pragma unroll
            for (int tp = 0; tp < 4; ++tp)
#pragma unroll
                for (int pp = 0; pp < 2; ++pp) lds128(a[2 * tp][pp], a[2 * tp + 1][pp], sA + c.offA[h][pp] + tp * 2048);
        } else {
#pragma unroll
            for (int u = 0; u < 8; ++u) lds128(a[u][0], a[u][1], sA + c.offA[h][0] + u * 8 * 128);
        }
        if (!TB) {
#pragma unroll
            for (int u = 0; u < 4; ++u) lds128(b[u][0], b[u][1], sB + c.offB[h][0] + u * 8 * 128);
        } else {
#pragma unroll
            for (int tp = 0; tp < 2; ++tp)
#pragma unroll
                for (int pp = 0; pp < 2; ++pp) lds128(b[2 * tp][pp], b[2 * tp + 1][pp], sB + c.offB[h][pp] + tp * 2048);
        }
        if (h == 1) {
            // all reads of this stage are issued; hand the slot back to the producer
            __syncwarp();
            if (c.lane == 0) mbar_arrive(ring.empty + 8 * stage);
        }
        if constexpr (S == Dmma::m8n8k4) {
#pragma unroll
            for (int pp = 0; pp < 2; ++pp)
#pragma unroll
                for (int i = 0; i < 8; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) dmma_m8n8k4(acc[i][j][0], acc[i][j][1], a[i][pp], b[j][pp]);
        } else {
#pragma unroll
            for (int pp = 0; pp < 2; ++pp)
#pragma unroll
                for (int i = 0; i < 8; i += 2)
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                        dmma_m16n8k4(acc[i][j][0], acc[i][j][1], acc[i + 1][j][0], acc[i + 1][j][1], a[i][pp], a[i + 1][pp],
                                     b[j][pp]);
        }
    }
}

// Row (A: slot x = r) or column (B: slot x = 2q + jj) inside the warp tile that MMA tile t of the accumulators holds,
// for an operand in MN form or in K form: the slot permutation of the fragment loads, undone.
template <bool MN>
__device__ __forceinline__ int tile_index(int t, int x) {
    return MN ? 16 * (t >> 1) + 2 * x + (t & 1) : 8 * t + perm8(x);
}

// Epilogue: stores this thread's accumulators of the tile at (m0, n0) into the M x N column-major D, combined with
// what D held or with an addend by op: D(m, n) = v after v = op.scale(acc) and op.add(v, col, m), where col =
// op.column(n) is the column the old values are read from (op.add2 combines rows m, m + 1 with one 16-byte read).
// vec allows 16-byte accesses: D and col 16-byte aligned with even leading dimensions.
template <bool TA, bool TB, class Op>
__device__ __forceinline__ void store_tile(const double (&acc)[8][4][2], const Consumer c, int m0, int n0, int M, int N,
                                           double* D, long long ldd, bool vec, const Op op) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {
            const int n = n0 + c.warp_n * 32 + tile_index<TB>(j, 2 * c.q + jj);
            if (n >= N) continue;
            double* dcol = D + (long long)n * ldd;
            const double* col = op.column(n);
            if (!TA) {
#pragma unroll
                for (int tp = 0; tp < 4; ++tp) {
                    const int m = m0 + c.warp_m * 64 + tile_index<true>(2 * tp, c.r);
                    if (m >= M) continue;
                    double v0 = op.scale(acc[2 * tp][j][jj]), v1 = op.scale(acc[2 * tp + 1][j][jj]);
                    if (vec && m + 1 < M) {
                        op.add2(v0, v1, col, m);
                        *reinterpret_cast<double2*>(dcol + m) = make_double2(v0, v1);
                    } else {
                        op.add(v0, col, m);
                        dcol[m] = v0;
                        if (m + 1 < M) {
                            op.add(v1, col, m + 1);
                            dcol[m + 1] = v1;
                        }
                    }
                }
            } else {
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int m = m0 + c.warp_m * 64 + tile_index<false>(i, c.r);
                    if (m >= M) continue;
                    double v = op.scale(acc[i][j][jj]);
                    op.add(v, col, m);
                    dcol[m] = v;
                }
            }
        }
    }
}

// C = alpha * acc + beta * C; C is not read when beta == 0.
struct ScaleAddC {
    const double* C;
    long long ldc;
    double alpha, beta;
    bool use_beta;
    __device__ __forceinline__ double scale(double a) const { return alpha * a; }
    __device__ __forceinline__ const double* column(int n) const { return C + (long long)n * ldc; }
    __device__ __forceinline__ void add(double& v, const double* col, int m) const {
        if (use_beta) v += beta * col[m];
    }
    __device__ __forceinline__ void add2(double& v0, double& v1, const double* col, int m) const {
        if (use_beta) {
            const double2 old = *reinterpret_cast<const double2*>(col + m);
            v0 += beta * old.x;
            v1 += beta * old.y;
        }
    }
};

// The persistent TMA + DMMA mainloop shared by the GEMM (SYRK = false: every tile of C, the whole K range, C = alpha*acc +
// beta*C) and the Gramian (SYRK = true: lower-triangle tiles only, split-K partials stored to a workspace).
template <Dmma S, bool TA, bool TB, bool SYRK>
__device__ __forceinline__ void dmma_persistent(const CUtensorMap& mapA, const CUtensorMap& mapB, const Params& p,
                                                const SyrkSched& sk) {
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int num_tiles = SYRK ? sk.tri_tiles * sk.splits : p.tiles_m * p.tiles_n;
    const int num_kb = (p.K + BK - 1) / BK;
    const Ring ring = ring_setup(&mapA, &mapB);

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
                    load_slab<TA, TB>(ring, stage, phase ^ 1, &mapA, &mapB, m0, n0, kb);
                    if (++stage == NUM_STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
        return;
    }

    // ========================= consumer warpgroups =========================
    setmaxnreg_inc<232>();
    const Consumer c = consumer_lane<TA, TB>(warp - 4, lane);
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

        double acc[8][4][2];
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;

        // bounded by p.K (a kernel parameter) rather than num_kb: one register fewer, which the <N,T> instance needs
        // to fit sm_90a's 168-register budget without a spill
        for (int k0 = k_begin; k0 < k_end; k0 += BK) {
            mma_slab<S, TA, TB>(acc, ring, stage, phase, c);
            if (++stage == NUM_STAGES) { stage = 0; phase ^= 1; }
        }

        store_tile<TA, TB>(acc, c, tm_ * BM, tn_ * BN, p.M, p.N, Cout, p.ldc, vec_ok,
                           ScaleAddC{Cout, p.ldc, p.alpha, p.beta, p.beta != 0.0});
    }
}

template <bool TA, bool TB>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_f64_dmma16x8_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
                         const Params p) {
    dmma_persistent<Dmma::m16n8k4, TA, TB, false>(mapA, mapB, p, SyrkSched{});
}

// Gramian partials: only the lower-triangle tiles of C = op(A) op(B) with op(B) = op(A)^T, split over K (see SyrkSched).
template <bool TA, bool TB>
__global__ void __launch_bounds__(NUM_THREADS, 1)
syrk_f64_dmma16x8_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
                         const Params p, const SyrkSched sk) {
    dmma_persistent<Dmma::m16n8k4, TA, TB, true>(mapA, mapB, p, sk);
}

// The m8n8k4 reference instances of the two (see the top of the file).
template <bool TA, bool TB>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_f64_dmma_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
                     const Params p) {
    dmma_persistent<Dmma::m8n8k4, TA, TB, false>(mapA, mapB, p, SyrkSched{});
}

template <bool TA, bool TB>
__global__ void __launch_bounds__(NUM_THREADS, 1)
syrk_f64_dmma_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
                     const Params p, const SyrkSched sk) {
    dmma_persistent<Dmma::m8n8k4, TA, TB, true>(mapA, mapB, p, sk);
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
//     st.global.v2.f64 go over NVLink.  Together: the GEMM epilogues do the reduce-scatter of the k partials;
//   * completion: when the last CTA tile of an entry whose output is local has been stored, one thread publishes a
//     local flag (st.release.sys) that the copy-out stream waits on.
// -------------------------------------------------------------------------------------------
struct G2Ent {
    double* D;
    const double* Cin;
    const unsigned long long* cin_flag;
    unsigned long long cin_val;
    unsigned long long* done_ctr;
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

// D = acc + Cin, or D = acc without an addend.  Cin is read with __ldcg: another GPU wrote it during this launch.
struct AddCin {
    const double* Cin;
    long long ldcin;
    __device__ __forceinline__ double scale(double a) const { return a; }
    __device__ __forceinline__ const double* column(int n) const { return Cin ? Cin + (long long)n * ldcin : nullptr; }
    __device__ __forceinline__ void add(double& v, const double* col, int m) const {
        if (col) v += __ldcg(col + m);
    }
    __device__ __forceinline__ void add2(double& v0, double& v1, const double* col, int m) const {
        if (col) {
            const double2 old = __ldcg(reinterpret_cast<const double2*>(col + m));
            v0 += old.x;
            v1 += old.y;
        }
    }
};

// D = Cin - acc (the Schur update C -= A B, with D == Cin allowed: every element is read and then written by the one
// thread that owns it).  One rounding, as in a GEMM into a temporary followed by an element-wise subtraction.
struct SubFromCin {
    const double* Cin;
    long long ldcin;
    __device__ __forceinline__ double scale(double a) const { return a; }
    __device__ __forceinline__ const double* column(int n) const { return Cin + (long long)n * ldcin; }
    __device__ __forceinline__ void add(double& v, const double* col, int m) const { v = __ldcg(col + m) - v; }
    __device__ __forceinline__ void add2(double& v0, double& v1, const double* col, int m) const {
        const double2 old = __ldcg(reinterpret_cast<const double2*>(col + m));
        v0 = old.x - v0;
        v1 = old.y - v1;
    }
};

// Epilogue op of a grouped launch: Op = AddCin (the blocked multiply and the multi-GPU protocol) or SubFromCin (every
// entry subtracts its product from Cin; gemm_f64_grouped2 picks this instance when the entries ask for it).
template <Dmma S, class Op>
__device__ __forceinline__ void dmma_grouped(const G2Params& g) {
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int num_tiles = g.num_tiles;
    const Ring ring = ring_setup(nullptr, nullptr);

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
                    const int nkb = en.nkb[sg];
                    for (int kb = 0; kb < nkb; ++kb) {
                        load_slab<false, false>(ring, stage, phase ^ 1, &g.mapA[ia], &g.mapB[ib], m0, n0, kb);
                        if (++stage == NUM_STAGES) { stage = 0; phase ^= 1; }
                    }
                }
            }
        }
        return;
    }

    setmaxnreg_inc<232>();
    const int cw = warp - 4;
    const Consumer cons = consumer_lane<false, false>(cw, lane);
    int stage = 0;
    uint32_t phase = 0;
    const unsigned long long* cin_seen = nullptr;      // last addend flag this thread has already observed
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        int c, tm_, tn_;
        locate(t, c, tm_, tn_);
        const G2Ent& en = g.e[c];
        int total_kb = 0;
        for (int sg = 0; sg < en.nseg; ++sg) total_kb += en.nkb[sg];
        double acc[8][4][2];
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;

        for (int kb = 0; kb < total_kb; ++kb) {
            mma_slab<S, false, false>(acc, ring, stage, phase, cons);
            if (++stage == NUM_STAGES) { stage = 0; phase ^= 1; }
        }

        // ---------------- epilogue: D = acc (+ Cin) ----------------
        double* D = en.D;
        const Op add{en.Cin, en.ldcin};
        const long long ldd = en.ldd;
        const int Mc = en.M, Nc = en.N;
        if (add.Cin != nullptr && en.cin_flag != nullptr && en.cin_flag != cin_seen) {
            // the other holder's partial must have landed in this GPU's staging buffer: lane 0 polls, then every other lane
            // acquires the flag through the same bounded wait (which returns on its first load).  Lane-dependent on purpose:
            // with one warp-uniform wait here nvcc 12.9 schedules the DMMA mainloop differently, and the 16384^2 grouped
            // multiply ran 18% slower (32.4 vs 39.3 TFLOP/s on an H100 80GB HBM3 at a 400 W power limit).
            const unsigned long long tag = (1ull << 56) | (3ull << 48) | (unsigned long long)c;
            if (lane == 0) wait_flag_ge<true>(en.cin_flag, en.cin_val, g.timeout_ns, g.status, tag);
            __syncwarp();
            if (lane != 0) wait_flag_ge<true>(en.cin_flag, en.cin_val, g.timeout_ns, g.status, tag);
            cin_seen = en.cin_flag;
        }
        const bool vec_ok = ((reinterpret_cast<uintptr_t>(D) & 15) == 0) && ((ldd & 1) == 0) &&
                            (add.Cin == nullptr || (((reinterpret_cast<uintptr_t>(add.Cin) & 15) == 0) && ((add.ldcin & 1) == 0)));
        // tile coordinates relative to the entry's region
        store_tile<false, false>(acc, cons, tm_ * BM, tn_ * BN, Mc, Nc, D, ldd, vec_ok, add);
        if (en.done_ctr != nullptr) {
            // The kernel only counts completion for entries whose output is LOCAL.  Every consumer thread fences its own
            // stores of this tile, the CTA barrier orders those fences before the count, then ONE thread counts the tile
            // and, if it was the entry's last, publishes the local flag with system scope (the copy-out stream polls it).
            // With the tile stored to a PEER GPU this sequence was measured faulty — one 16x32 patch of a tile stale in
            // about a third of the 8192^2 calls — so csrc/dist.cu announces peer outputs after the launch with a stream
            // memory operation (two-launch reduce-scatter) or pushes them with the copy engine (host path).
            __threadfence_system();
            asm volatile("bar.sync 1, %0;" ::"n"(NUM_CONSUMER_WARPS * 32) : "memory");
            if (cw == 0 && lane == 0) {
                __threadfence_system();
                const unsigned long long prev = atomicAdd(en.done_ctr, 1ull);
                if (prev + 1ull == (unsigned long long)(en.tiles_m * en.tiles_n)) {
                    __threadfence_system();
                    if (en.sig_local) asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(en.sig_local), "l"(en.sig_val) : "memory");
                }
            }
        }
    }
}

__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_f64_dmma16x8_grouped_kernel(const __grid_constant__ G2Params g) {
    dmma_grouped<Dmma::m16n8k4, AddCin>(g);
}

// The m8n8k4 reference instance (see the top of the file).
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_f64_dmma_grouped_kernel(const __grid_constant__ G2Params g) {
    dmma_grouped<Dmma::m8n8k4, AddCin>(g);
}

// D = Cin - acc for every entry (mb_block_schur_update), and its m8n8k4 reference instance.
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_f64_dmma16x8_grouped_sub_kernel(const __grid_constant__ G2Params g) {
    dmma_grouped<Dmma::m16n8k4, SubFromCin>(g);
}
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_f64_dmma_grouped_sub_kernel(const __grid_constant__ G2Params g) {
    dmma_grouped<Dmma::m8n8k4, SubFromCin>(g);
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

// How the DMMA kernels stage an fp64 operand that is mn x k in the product (mn = M for A, N for B).
enum class Form {
    MN,   // stored mn x k, mn contiguous: 8 boxes of [16 k][16 mn] per slab (A 'N', B 'T')
    K,    // stored k x mn, k contiguous: one box of [128 mn][16 k] per slab (A 'T', B 'N')
};

bool operand_map(CUtensorMap* map, const double* base, int mn, int k, long long ld, Form form) {
    return form == Form::MN ? tma_map(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, base, mn, k, ld * 8, 16, 16)
                            : tma_map(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, base, k, mn, ld * 8, 16, 128);
}

template <bool TA, bool TB>
cudaError_t launch_gemm(int grid, cudaStream_t stream, const CUtensorMap& mA, const CUtensorMap& mB, const Params& p) {
    return g_call.dmma_reference
               ? launch_with_smem<gemm_f64_dmma_kernel<TA, TB>>(grid, NUM_THREADS, SMEM_BYTES, stream, mA, mB, p)
               : launch_with_smem<gemm_f64_dmma16x8_kernel<TA, TB>>(grid, NUM_THREADS, SMEM_BYTES, stream, mA, mB, p);
}

template <bool TA, bool TB>
cudaError_t launch_syrk(int grid, cudaStream_t stream, const CUtensorMap& mA, const Params& p, const SyrkSched& sk) {
    return g_call.dmma_reference
               ? launch_with_smem<syrk_f64_dmma_kernel<TA, TB>>(grid, NUM_THREADS, SMEM_BYTES, stream, mA, mA, p, sk)
               : launch_with_smem<syrk_f64_dmma16x8_kernel<TA, TB>>(grid, NUM_THREADS, SMEM_BYTES, stream, mA, mA, p, sk);
}

}  // namespace

bool gemm_f64_tma_eligible(const double* A, long long lda, const double* B, long long ldb) {
    return ((reinterpret_cast<uintptr_t>(A) & 15) == 0) && ((reinterpret_cast<uintptr_t>(B) & 15) == 0) &&
           (lda % 2 == 0) && (ldb % 2 == 0) && tma_encode_fn() != nullptr;
}

cudaError_t gemm_f64(bool transA, bool transB, int M, int N, int K, double alpha, const double* A, long long lda,
                     const double* B, long long ldb, double beta, double* C, long long ldc, int num_sms,
                     cudaStream_t stream, bool force_generic) {
    if (M <= 0 || N <= 0) return cudaSuccess;
    if (K <= 0 || alpha == 0.0) {
        if (beta == 1.0) return cudaSuccess;
        scale_matrix_kernel<<<min(1184, (int)(((long long)M * N + 255) / 256)), 256, 0, stream>>>(M, N, beta, C, ldc);
        return launched();
    }
    if (!force_generic && gemm_f64_tma_eligible(A, lda, B, ldb)) {
        CUtensorMap mA, mB;
        if (operand_map(&mA, A, M, K, lda, transA ? Form::K : Form::MN) &&
            operand_map(&mB, B, N, K, ldb, transB ? Form::MN : Form::K)) {
            Params p;
            p.M = M; p.N = N; p.K = K; p.alpha = alpha; p.beta = beta; p.C = C; p.ldc = ldc;
            p.tiles_m = (M + BM - 1) / BM;
            p.tiles_n = (N + BN - 1) / BN;
            const int grid = min(p.tiles_m * p.tiles_n, num_sms);
            if (!transA && !transB) return launch_gemm<false, false>(grid, stream, mA, mB, p);
            if (transA && !transB) return launch_gemm<true, false>(grid, stream, mA, mB, p);
            if (!transA && transB) return launch_gemm<false, true>(grid, stream, mA, mB, p);
            return launch_gemm<true, true>(grid, stream, mA, mB, p);
        }
    }
    dim3 grid((M + 63) / 64, (N + 63) / 64);
    if (!transA && !transB)
        gemm_f64_generic_kernel<false, false><<<grid, 256, 0, stream>>>(M, N, K, alpha, A, lda, B, ldb, beta, C, ldc);
    else if (transA && !transB)
        gemm_f64_generic_kernel<true, false><<<grid, 256, 0, stream>>>(M, N, K, alpha, A, lda, B, ldb, beta, C, ldc);
    else if (!transA && transB)
        gemm_f64_generic_kernel<false, true><<<grid, 256, 0, stream>>>(M, N, K, alpha, A, lda, B, ldb, beta, C, ldc);
    else
        gemm_f64_generic_kernel<true, true><<<grid, 256, 0, stream>>>(M, N, K, alpha, A, lda, B, ldb, beta, C, ldc);
    return launched();
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
                     int num_sms, cudaStream_t stream) {
    if (n <= 0) return cudaSuccess;
    // op(A) and op(A)^T are read from the same storage in the same form, so A and B share one map
    CUtensorMap mA;
    const bool tma = K > 0 && gemm_f64_tma_eligible(A, lda, A, lda) && operand_map(&mA, A, n, K, lda, trans ? Form::K : Form::MN);
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
        const int grid = min(sk.tri_tiles * splits, num_sms);
        e = !trans ? launch_syrk<false, true>(grid, stream, mA, p, sk) : launch_syrk<true, false>(grid, stream, mA, p, sk);
        if (e != cudaSuccess) return e;
    } else {
        // the whole product on the CUDA cores (views TMA cannot address), or zeros for K = 0
        e = gemm_f64(trans, !trans, n, n, K, 1.0, A, lda, A, lda, 0.0, P, ldp, num_sms, stream, true);
        if (e != cudaSuccess) return e;
    }
    const int nb = (n + 31) / 32;
    const unsigned grid = nb * (nb + 1) / 2;
    if (((reinterpret_cast<uintptr_t>(P) & 15) == 0) && ((ldp & 1) == 0))
        gram_reduce_mirror_kernel<true><<<grid, 256, 0, stream>>>(P, ldp, ldp * n, splits, n, G, ldg);
    else
        gram_reduce_mirror_kernel<false><<<grid, 256, 0, stream>>>(P, ldp, ldp * n, splits, n, G, ldg);
    return launched();
}

cudaError_t gemm_f64_grouped2(const G2Launch& L, int num_sms, cudaStream_t stream) {
    if (L.ne <= 0) return cudaSuccess;
    if (L.ne > G2_MAX_ENTRIES || L.na > G2_MAX_OPS || L.nb > G2_MAX_OPS || !tma_encode_fn()) return cudaErrorNotSupported;
    static thread_local G2Params g;          // ~20 KB parameter block: kept off the stack, one per calling thread
    for (int i = 0; i < L.na; ++i) {
        const G2Operand& o = L.A[i];
        if (o.rows <= 0 || o.cols <= 0 || !gemm_f64_tma_eligible(o.ptr, o.ld, o.ptr, 2)) return cudaErrorNotSupported;
        if (!operand_map(&g.mapA[i], o.ptr, o.rows, o.cols, o.ld, Form::MN)) return cudaErrorNotSupported;
        if (o.ready_base >= 0 && (o.band <= 0 || o.band % BM != 0)) return cudaErrorInvalidValue;
        g.a_band[i] = o.band > 0 ? o.band : (1 << 30);
        g.a_ready[i] = (short)o.ready_base;
    }
    for (int i = 0; i < L.nb; ++i) {
        const G2Operand& o = L.B[i];
        if (o.rows <= 0 || o.cols <= 0 || !gemm_f64_tma_eligible(o.ptr, o.ld, o.ptr, 2)) return cudaErrorNotSupported;
        if (!operand_map(&g.mapB[i], o.ptr, o.cols, o.rows, o.ld, Form::K)) return cudaErrorNotSupported;
        if (o.ready_base >= 0 && (o.band <= 0 || o.band % BN != 0)) return cudaErrorInvalidValue;
        g.b_band[i] = o.band > 0 ? o.band : (1 << 30);
        g.b_ready[i] = (short)o.ready_base;
    }
    int tiles = 0;
    const bool sub = L.E[0].sub_from_cin;
    for (int c = 0; c < L.ne; ++c) {
        const G2Entry& s = L.E[c];
        G2Ent& d = g.e[c];
        if (s.nseg <= 0 || s.nseg > G2_MAX_SEG || s.M <= 0 || s.N <= 0) return cudaErrorNotSupported;
        if (s.sub_from_cin != sub || (sub && (s.Cin == nullptr || s.cin_flag != nullptr))) return cudaErrorInvalidValue;
        if ((s.m_off % BM) != 0 || (s.n_off % BN) != 0) return cudaErrorInvalidValue;
        d.D = s.D; d.ldd = s.ldd; d.Cin = s.Cin; d.ldcin = s.ldcin;
        d.cin_flag = s.cin_flag; d.cin_val = s.cin_val;
        d.done_ctr = s.done_ctr; d.sig_local = s.sig_local; d.sig_val = s.sig_val;
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
    const int grid = min(tiles, num_sms);
    if (sub)
        return g_call.dmma_reference
                   ? launch_with_smem<gemm_f64_dmma_grouped_sub_kernel>(grid, NUM_THREADS, SMEM_BYTES, stream, g)
                   : launch_with_smem<gemm_f64_dmma16x8_grouped_sub_kernel>(grid, NUM_THREADS, SMEM_BYTES, stream, g);
    return g_call.dmma_reference
               ? launch_with_smem<gemm_f64_dmma_grouped_kernel>(grid, NUM_THREADS, SMEM_BYTES, stream, g)
               : launch_with_smem<gemm_f64_dmma16x8_grouped_kernel>(grid, NUM_THREADS, SMEM_BYTES, stream, g);
}

cudaError_t gemm_f64_grouped(int m, int k, int n, const int* my_c, int num_c, const double* const* A, const long long* lda,
                             const double* const* B, const long long* ldb, double* const* C, const long long* ldc,
                             const int* row_len, const int* k_len, const int* col_len, int num_sms, cudaStream_t stream) {
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
    return gemm_f64_grouped2(L, num_sms, stream);
}

}  // namespace mb

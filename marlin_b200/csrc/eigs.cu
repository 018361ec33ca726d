// y = A^T (A x) for a row-major fp64 view, reading each row from HBM once where it fits (multiplyGramianMatrixBy,
// matrix/DenseVecMatrix.scala:1444-1459: sum over the rows of (a_r . x) a_r).
//
// gm_tile_kernel: a persistent CTA owns tiles of R rows (tiles blockIdx.x, blockIdx.x + gridDim.x, ...), three roles:
//   warp 0       producer: each lane streams one row of a tile piece into a GM_STAGES-deep ring of shared-memory stages
//                with one plain bulk copy (cp.async.bulk, completing on the stage's mbarrier), so any ld and any 8-byte
//                alignment is read in place.
//   warps 1-4    phase 1: t_r = a_r . x, one warp per row: lane l sums the columns l, l + 32, ... of each piece in
//                ascending order, then the 32 lane sums are added by a fixed xor butterfly.
//   warps 5-8    phase 2: y_part[j] += t_r * a_rj over the tile's rows in ascending order, one thread per column.
// The two groups hand the tile over through a double-buffered t (mbarriers tfull / tempty), so phase 1 of tile q + 1
// runs while phase 2 of tile q does.  Every multiply and add is a separate DMUL / DADD (no DFMA).
//
// Resident tiles (n <= GM_STAGE - 2 = 5118): R = min(32, GM_STAGE / slot) whole rows per stage; phase 2 reads them where
// phase 1 did, and y_part lives in shared memory.  HBM bytes per product: 8 m n for A.
// Wide tiles (n > 5118): R = 8 rows in pieces of GM_WIDE_CW = 638 columns.  Each phase has its own two stages; phase 2
// streams the pieces of tile q again while phase 1 streams those of tile q + 1; y_part is the CTA's row of `part` in
// global memory.  Between the two reads of a piece each SM streams about two tiles (128 n bytes); 132 SMs keep that in
// H100's 50 MB L2 only up to n of about 3000, which resident tiles already cover, so every wide re-read comes from HBM:
// 16 m n bytes for A, plus 16 n ceil(m / 8) bytes of y_part traffic (mostly L2).
// gm_fold_kernel sums the CTAs' partials in ascending CTA order (8 n grid bytes besides x and y).  No atomics: the same
// inputs give the same bits on every run.
#include "eigs.h"
#include "ptx.cuh"
#include "launch.h"

#include <cstdint>

namespace mb {
namespace {

constexpr int GM_THREADS = 288;              // producer warp + two groups of four warps
constexpr int GM_STAGES = 4;
constexpr int GM_STAGE = 5120;               // doubles per stage (40 KiB)
constexpr int GM_MAX_ROWS = 32;              // one producer lane per row
constexpr int GM_WIDE_ROWS = 8;
constexpr int GM_WIDE_CW = GM_STAGE / GM_WIDE_ROWS - 2;
constexpr int GM_RESIDENT_N = GM_STAGE - 2;
constexpr int GM_SMEM = (2 * GM_STAGES + 4) * 8 + 2 * GM_MAX_ROWS * 8 + GM_STAGES * GM_STAGE * 8 + GM_STAGE * 8;

struct GmShape {
    const double* a;
    long long ld;
    long long m;
    int n;
    const double* x;
    long long incx;
    int rows;         // R
    int slot;         // doubles per row slot
    int cw;           // columns per piece
    int nch;          // pieces per row
    long long ntiles;
    bool resident;
};

__device__ __forceinline__ void group_sync(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

__device__ __forceinline__ void gm_wait(const uint64_t* bar, long long use) {
    mbar_wait(smem_u32(bar), static_cast<uint32_t>(use & 1));
}

__global__ void __launch_bounds__(GM_THREADS, 1) gm_tile_kernel(GmShape s, double* part) {
    extern __shared__ __align__(16) unsigned char gm_smem[];
    uint64_t* full = reinterpret_cast<uint64_t*>(gm_smem);
    uint64_t* empty = full + GM_STAGES;
    uint64_t* tfull = empty + GM_STAGES;
    uint64_t* tempty = tfull + 2;
    double* tb = reinterpret_cast<double*>(tempty + 2);            // [2][GM_MAX_ROWS]
    double* ring = tb + 2 * GM_MAX_ROWS;
    double* ys = ring + GM_STAGES * GM_STAGE;                      // y_part of a resident shape
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        for (int i = 0; i < GM_STAGES; ++i) {
            mbar_init(smem_u32(&full[i]), 1);
            mbar_init(smem_u32(&empty[i]), 1);
        }
        for (int i = 0; i < 2; ++i) {
            mbar_init(smem_u32(&tfull[i]), 1);
            mbar_init(smem_u32(&tempty[i]), 1);
        }
        fence_barrier_init();
    }
    __syncthreads();
    const long long grid = gridDim.x;
    // Which stage a piece uses, and its use count there.  Resident: one ring of GM_STAGES whole tiles that both phases
    // read.  Wide: phase 1 and phase 2 each have a ring of GM_STAGES / 2 and read every piece of their own ring in order,
    // so no waiter is ever two barrier phases behind.
    auto place = [&](long long q, int c, bool second, int* stage, long long* use) {
        if (s.resident) {
            *stage = static_cast<int>(q % GM_STAGES);
            *use = q / GM_STAGES;
        } else {
            const long long i = q * s.nch + c;
            *stage = static_cast<int>(i % (GM_STAGES / 2)) + (second ? GM_STAGES / 2 : 0);
            *use = i / (GM_STAGES / 2);
        }
    };
    if (warp == 0) {
        // ---- producer: piece c of tile q (for phase 2 if `second`) once its stage's previous use is released.  Wide
        // tiles go p1(0), then p2(q) and p1(q + 1) piece by piece, so both phases keep streaming.
        auto issue = [&](long long q, int c, bool second) {
            const long long t = blockIdx.x + q * grid;
            int stage;
            long long use;
            place(q, c, second, &stage, &use);
            if (use > 0) gm_wait(&empty[stage], use - 1);
            const long long r0 = t * s.rows;
            const int nr = static_cast<int>(min((long long)s.rows, s.m - r0));
            const long long c0 = (long long)c * s.cw;
            const int cw = static_cast<int>(min((long long)s.cw, s.n - c0));
            uint32_t bytes = 0;
            int lead = 0;
            const double* src = nullptr;
            if (lane < nr) src = piece_span(s.a + (r0 + lane) * s.ld + c0, cw, &bytes, &lead);
            const uint32_t total = __reduce_add_sync(0xffffffffu, bytes);
            const uint32_t bar = smem_u32(&full[stage]);
            if (lane == 0) mbar_arrive_expect_tx(bar, total);
            __syncwarp();
            if (lane < nr) bulk_load(smem_u32(ring + (long long)stage * GM_STAGE + lane * s.slot), src, bytes, bar);
        };
        auto exists = [&](long long q) { return blockIdx.x + q * grid < s.ntiles; };
        if (s.resident) {
            for (long long q = 0; exists(q); ++q) issue(q, 0, false);
        } else {
            for (int c = 0; c < s.nch; ++c) issue(0, c, false);
            for (long long q = 0; exists(q); ++q)
                for (int c = 0; c < s.nch; ++c) {
                    issue(q, c, true);
                    if (exists(q + 1)) issue(q + 1, c, false);
                }
        }
    } else if (warp <= 4) {
        // ---- phase 1: t_r = a_r . x
        const int g = tid - 32, w = g >> 5;
        for (long long q = 0;; ++q) {
            const long long t = blockIdx.x + q * grid;
            if (t >= s.ntiles) break;
            const long long r0 = t * s.rows;
            const int nr = static_cast<int>(min((long long)s.rows, s.m - r0));
            double acc[GM_MAX_ROWS / 4];
#pragma unroll
            for (int i = 0; i < GM_MAX_ROWS / 4; ++i) acc[i] = 0.0;
            for (int c = 0; c < s.nch; ++c) {
                int stage;
                long long use;
                place(q, c, false, &stage, &use);
                gm_wait(&full[stage], use);
                const long long c0 = (long long)c * s.cw;
                const int cw = static_cast<int>(min((long long)s.cw, s.n - c0));
                const double* xc = s.x + c0 * s.incx;
#pragma unroll
                for (int i = 0; i < GM_MAX_ROWS / 4; ++i) {
                    const int r = w + 4 * i;
                    if (r < nr) {
                        const double* row = ring + stage * GM_STAGE + r * s.slot + piece_lead(s.a + (r0 + r) * s.ld + c0);
                        double v = acc[i];
                        for (int j = lane; j < cw; j += 32) v = __dadd_rn(v, __dmul_rn(row[j], __ldg(xc + j * s.incx)));
                        acc[i] = v;
                    }
                }
                if (!s.resident) {
                    group_sync(1);
                    if (g == 0) mbar_arrive(smem_u32(&empty[stage]));
                }
            }
            if (q >= 2) gm_wait(&tempty[q & 1], (q >> 1) - 1);
#pragma unroll
            for (int i = 0; i < GM_MAX_ROWS / 4; ++i) {
                double v = acc[i];
#pragma unroll
                for (int o = 16; o >= 1; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
                const int r = w + 4 * i;
                if (lane == 0 && r < nr) tb[(q & 1) * GM_MAX_ROWS + r] = v;
            }
            group_sync(1);
            if (g == 0) mbar_arrive(smem_u32(&tfull[q & 1]));
        }
    } else {
        // ---- phase 2: y_part += t_r a_r, rows ascending
        const int g = tid - 160;
        double* y = s.resident ? ys : part + (long long)blockIdx.x * s.n;
        for (long long j = g; j < s.n; j += 128) y[j] = 0.0;
        for (long long q = 0;; ++q) {
            const long long t = blockIdx.x + q * grid;
            if (t >= s.ntiles) break;
            const long long r0 = t * s.rows;
            const int nr = static_cast<int>(min((long long)s.rows, s.m - r0));
            const double* tq = tb + (q & 1) * GM_MAX_ROWS;
            gm_wait(&tfull[q & 1], q >> 1);
            for (int c = 0; c < s.nch; ++c) {
                int stage;
                long long use;
                place(q, c, true, &stage, &use);
                gm_wait(&full[stage], use);                // complete already for a resident tile; makes the bytes visible
                const long long c0 = (long long)c * s.cw;
                const int cw = static_cast<int>(min((long long)s.cw, s.n - c0));
                const double* st = ring + stage * GM_STAGE;
                // row r starts (lead0 + r * ld) & 1 doubles into its slot: the rows are 8-byte aligned
                const int lead0 = piece_lead(s.a + r0 * s.ld + c0), ldodd = static_cast<int>(s.ld & 1);
                for (int j = g; j < cw; j += 128) {
                    double v = y[c0 + j];
                    for (int r = 0; r < nr; ++r)
                        v = __dadd_rn(v, __dmul_rn(tq[r], st[r * s.slot + ((lead0 + r * ldodd) & 1) + j]));
                    y[c0 + j] = v;
                }
                group_sync(2);
                if (g == 0) {
                    mbar_arrive(smem_u32(&empty[stage]));
                    if (c == s.nch - 1) mbar_arrive(smem_u32(&tempty[q & 1]));
                }
            }
        }
        if (s.resident) {
            double* out = part + (long long)blockIdx.x * s.n;
            for (long long j = g; j < s.n; j += 128) out[j] = ys[j];
        }
    }
}

// y[j] = part[0][j] + part[1][j] + ... (ascending), then + y[j] when accumulating; nparts = 0 gives 0.
__global__ void __launch_bounds__(256) gm_fold_kernel(const double* part, int nparts, int n, double* y, long long incy,
                                                      bool accumulate) {
    const long long j = (long long)blockIdx.x * 256 + threadIdx.x;
    if (j >= n) return;
    double s = nparts ? part[j] : 0.0;
    for (int p = 1; p < nparts; ++p) s = __dadd_rn(s, part[(long long)p * n + j]);
    y[j * incy] = accumulate ? __dadd_rn(y[j * incy], s) : s;
}

GmShape gm_shape(long long m, int n) {
    GmShape s{};
    s.m = m;
    s.n = n;
    s.resident = n <= GM_RESIDENT_N;
    if (s.resident) {
        s.slot = (n + 2) & ~1;                 // a row's 16-byte-aligned span is at most n + 1 doubles, kept even
        s.rows = GM_STAGE / s.slot < GM_MAX_ROWS ? GM_STAGE / s.slot : GM_MAX_ROWS;
        s.cw = n;
        s.nch = 1;
    } else {
        s.rows = GM_WIDE_ROWS;
        s.slot = GM_WIDE_CW + 2;
        s.cw = GM_WIDE_CW;
        s.nch = (int)(((long long)n + GM_WIDE_CW - 1) / GM_WIDE_CW);
    }
    s.ntiles = (m + s.rows - 1) / s.rows;
    return s;
}

}  // namespace

int gram_matvec_parts(long long m, int n, int num_sms) {
    if (m <= 0 || n <= 0) return 0;
    const long long tiles = gm_shape(m, n).ntiles;
    return (int)(tiles < num_sms ? tiles : num_sms);
}

cudaError_t gram_matvec_f64(const double* a, long long lda, long long m, int n, const double* x, long long incx, double* y,
                            long long incy, bool accumulate, double* part, int num_sms, cudaStream_t st) {
    if (n <= 0 || m < 0) return n == 0 ? cudaSuccess : cudaErrorInvalidValue;
    const int grid = gram_matvec_parts(m, n, num_sms);
    if (grid > 0) {
        GmShape s = gm_shape(m, n);
        s.a = a;
        s.ld = lda;
        s.x = x;
        s.incx = incx;
        const cudaError_t e = launch_with_smem<gm_tile_kernel>(grid, GM_THREADS, GM_SMEM, st, s, part);
        if (e != cudaSuccess) return e;
    } else if (accumulate) {
        return cudaSuccess;
    }
    gm_fold_kernel<<<(unsigned)(((long long)n + 255) / 256), 256, 0, st>>>(part, grid, n, y, incy, accumulate);
    return launched();
}

}  // namespace mb

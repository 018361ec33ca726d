// One step of DenseVecMatrix.lr (matrix/DenseVecMatrix.scala:1005-1035) over a row-major fp64 shard:
//   margin_r = -(x~_r . w),  g_r = 1 / (1 + exp(margin_r)) - x_r0,  delta = sum_r x~_r * g_r,  w -= delta * scale
// where x~_r is row r with element 0 (the label) replaced by the intercept 1.
//
// lr_grad_tile_kernel: a persistent CTA owns tiles of LR_ROWS rows (tiles blockIdx.x, blockIdx.x + gridDim.x, ...).
// Warp 0 streams each row in LR_CHUNK-column pieces into a shared-memory ring with plain bulk copies (one
// cp.async.bulk per row piece, completing on the stage's mbarrier), so any ld and any 8-byte alignment is read in place.
//   phase 1  warp 0, one lane per row: the margin, sequential in column order with separate multiplies and adds --
//            bit for bit BLAS ddot as F2J runs it (oracle mo_ddot_f2j) -- then g_r.
//   phase 2  all 128 threads, one column each: acc_j += x~_rj * g_r over the tile's rows in ascending order, into the
//            CTA's partial gradient part[blockIdx.x][j] (each column always belongs to the same thread).
// When a tile's row pieces fit in half the ring (n <= LR_STAGES / 2 * LR_CHUNK = 384 columns) phase 2 reads them where
// phase 1 left them and the next tile streams in meanwhile: the shard crosses HBM once.  Wider rows are streamed a second
// time for phase 2, right after phase 1 of the same 32 rows; that re-read is served by L2 while the CTAs' tiles in flight,
// 132 x 32 x n x 8 bytes, fit in it (about n = 1500 on H100's 50 MB).
// lr_fold_kernel sums the partials in ascending CTA order and either writes the sum or applies the update.
// Everything is deterministic: the same inputs give the same bits on every run.
#include "logistic.h"
#include "ptx.cuh"
#include "launch.h"

#include <cstdint>

namespace mb {
namespace {

constexpr int LR_ROWS = 32;                  // rows per tile: one margin chain per lane of warp 0
constexpr int LR_THREADS = 128;
constexpr int LR_CHUNK = 128;                // columns per row piece (one per thread in phase 2)
constexpr int LR_SLOT = LR_CHUNK + 2;        // doubles per row slot: a piece plus its 16-byte alignment lead and tail
constexpr int LR_STAGES = 6;
constexpr int LR_STAGE_DOUBLES = LR_ROWS * LR_SLOT;
constexpr int LR_SMEM = LR_STAGES * LR_STAGE_DOUBLES * 8 + LR_STAGES * 8 + LR_ROWS * 8;

struct LrShape {
    const double* x;
    long long ld;
    int m, n;
    int nch;          // row pieces per row
    int per_tile;     // loads per tile: nch, or 2 * nch when phase 2 streams the tile again
    int ntiles;
};

// Warp 0 (all lanes): issue load k of this CTA's sequence into stage k % LR_STAGES, if it exists.
__device__ __forceinline__ void lr_issue(const LrShape& s, int k, double* ring, uint64_t* full) {
    const int q = k / s.per_tile;
    const int c = (k % s.per_tile) % s.nch;
    const long long t = blockIdx.x + (long long)q * gridDim.x;
    if (t >= s.ntiles) return;
    const int lane = threadIdx.x & 31;
    const long long r0 = t * LR_ROWS;
    const int nr = static_cast<int>(min((long long)LR_ROWS, s.m - r0));
    const int c0 = c * LR_CHUNK, cw = min(LR_CHUNK, s.n - c0);
    const int stage = k % LR_STAGES;
    uint32_t bytes = 0;
    int lead = 0;
    const double* src = nullptr;
    if (lane < nr) src = piece_span(s.x + (r0 + lane) * s.ld + c0, cw, &bytes, &lead);
    const uint32_t total = __reduce_add_sync(0xffffffffu, bytes);
    const uint32_t bar = smem_u32(&full[stage]);
    if (lane == 0) mbar_arrive_expect_tx(bar, total);
    __syncwarp();
    if (lane < nr) bulk_load(smem_u32(ring + (long long)stage * LR_STAGE_DOUBLES + lane * LR_SLOT), src, bytes, bar);
}

// gradientMul = 1 / (1 + exp(-1.0 * dot)) - label.  exp and the correctly rounded division are built on DFMA; keeping them
// out of line keeps every multiply and add of the kernel's own arithmetic a separate DMUL / DADD (checked in the SASS).
__device__ __noinline__ double lr_gradient_mul(double dot, double label) {
    const double margin = __dmul_rn(-1.0, dot);
    return __dsub_rn(__ddiv_rn(1.0, __dadd_rn(1.0, exp(margin))), label);
}

__device__ __forceinline__ void lr_wait(const uint64_t* full, int k) {
    mbar_wait(smem_u32(&full[k % LR_STAGES]), static_cast<uint32_t>((k / LR_STAGES) & 1));
}

__global__ void __launch_bounds__(LR_THREADS, 1) lr_grad_tile_kernel(LrShape s, const double* __restrict__ w, double* part) {
    extern __shared__ __align__(16) unsigned char lr_smem[];
    double* ring = reinterpret_cast<double*>(lr_smem);
    uint64_t* full = reinterpret_cast<uint64_t*>(ring + LR_STAGES * LR_STAGE_DOUBLES);
    double* gs = reinterpret_cast<double*>(full + LR_STAGES);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    double* mypart = part + (long long)blockIdx.x * s.n;
    for (int j = tid; j < s.n; j += LR_THREADS) mypart[j] = 0.0;
    if (tid == 0) {
        for (int i = 0; i < LR_STAGES; ++i) mbar_init(smem_u32(&full[i]), 1);
        fence_barrier_init();
    }
    __syncthreads();
    if (warp == 0)
        for (int k = 0; k < LR_STAGES; ++k) lr_issue(s, k, ring, full);
    const bool resident = s.per_tile == s.nch;
    int kbase = 0;
    for (int t = blockIdx.x; t < s.ntiles; t += gridDim.x, kbase += s.per_tile) {
        const long long r0 = (long long)t * LR_ROWS;
        const int nr = static_cast<int>(min((long long)LR_ROWS, s.m - r0));
        if (warp == 0) {
            // phase 1: lane = row
            const double* row = s.x + (r0 + lane) * s.ld;
            double dot = 0.0, label = 0.0;
            for (int c = 0; c < s.nch; ++c) {
                const int k = kbase + c;
                lr_wait(full, k);
                const int c0 = c * LR_CHUNK, cw = min(LR_CHUNK, s.n - c0);
                if (lane < nr) {
                    const double* xs = ring + (k % LR_STAGES) * LR_STAGE_DOUBLES + lane * LR_SLOT + piece_lead(row + c0);
                    const double* wc = w + c0;
                    int j = 0;
                    if (c == 0) {
                        label = xs[0];
                        dot = __dadd_rn(dot, __dmul_rn(1.0, __ldg(wc)));          // the intercept replaces the label
                        j = 1;
                    }
#pragma unroll 8
                    for (; j < cw; ++j) dot = __dadd_rn(dot, __dmul_rn(xs[j], __ldg(wc + j)));
                }
                if (!resident) {
                    __syncwarp();
                    lr_issue(s, k + LR_STAGES, ring, full);
                }
            }
            if (lane < nr) gs[lane] = lr_gradient_mul(dot, label);
        }
        __syncthreads();
        // phase 2: thread = column of the piece
        for (int c = 0; c < s.nch; ++c) {
            const int k = kbase + (resident ? 0 : s.nch) + c;
            const int c0 = c * LR_CHUNK, cw = min(LR_CHUNK, s.n - c0);
            double acc = tid < cw ? mypart[c0 + tid] : 0.0;
            lr_wait(full, k);                // already complete for a resident tile; the wait makes the bytes visible here
            if (tid < cw) {
                const double* xs = ring + (k % LR_STAGES) * LR_STAGE_DOUBLES + tid;
                const double* row = s.x + r0 * s.ld + c0;
                const bool icpt = c0 + tid == 0;
                for (int r = 0; r < nr; ++r, row += s.ld) {
                    const double v = icpt ? 1.0 : xs[r * LR_SLOT + piece_lead(row)];
                    acc = __dadd_rn(acc, __dmul_rn(v, gs[r]));
                }
                mypart[c0 + tid] = acc;
            }
            __syncthreads();                 // the stage and (after the last piece) gs are free again
            if (warp == 0) {
                fence_proxy_async();
                lr_issue(s, k + LR_STAGES, ring, full);
            }
        }
    }
}

// out[j] = part[0][j] + part[1][j] + ... (ascending), or w[j] -= that * scale
__global__ void __launch_bounds__(256) lr_fold_kernel(const double* part, int nparts, int n, double* out, double* w, double scale) {
    const int j = blockIdx.x * 256 + threadIdx.x;
    if (j >= n) return;
    double s = part[j];
    for (int p = 1; p < nparts; ++p) s = __dadd_rn(s, part[(long long)p * n + j]);
    if (w)
        w[j] = __dsub_rn(w[j], __dmul_rn(s, scale));
    else
        out[j] = s;
}

}  // namespace

int lr_parts(int m, int num_sms) {
    const long long tiles = ((long long)m + LR_ROWS - 1) / LR_ROWS;
    return (int)(tiles < 1 ? 1 : (tiles < num_sms ? tiles : num_sms));
}

cudaError_t lr_gradient_f64(const double* x, long long ld, int m, int n, double* w, double* part, double* out, bool update,
                            double scale, int num_sms, cudaStream_t st) {
    if (m <= 0 || n <= 0) return cudaErrorInvalidValue;
    LrShape s;
    s.x = x;
    s.ld = ld;
    s.m = m;
    s.n = n;
    s.nch = (n + LR_CHUNK - 1) / LR_CHUNK;
    s.per_tile = 2 * s.nch <= LR_STAGES ? s.nch : 2 * s.nch;
    s.ntiles = (int)(((long long)m + LR_ROWS - 1) / LR_ROWS);
    const int grid = lr_parts(m, num_sms);
    cudaError_t e = launch_with_smem<lr_grad_tile_kernel>(grid, LR_THREADS, LR_SMEM, st, s, (const double*)w, part);
    if (e != cudaSuccess) return e;
    lr_fold_kernel<<<(n + 255) / 256, 256, 0, st>>>(part, grid, n, update ? nullptr : out, update ? w : nullptr, scale);
    return launched();
}

}  // namespace mb

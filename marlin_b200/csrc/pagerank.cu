// PageRank (examples/PageRank.scala): one iteration `links.multiply(ranks)`, `.reduce(add)`, `.add(0.15 * ones)` over the
// in-link CSR of the link matrix (rows = target pages, columns = ascending source pages, values fl(fl(1 / size) * 0.85)).
//
// Arithmetic of row i: P_s = 0.0 + fl(w_i,j0 * x_j0) + fl(w_i,j1 * x_j1) + ... over the stored sources j of segment s
// (sources [s * seg_len, (s + 1) * seg_len)) in ascending order, each multiply and add rounded separately (__dmul_rn /
// __dadd_rn, no DFMA); y_i = fl(fl(0.0 + P_0 + P_1 + ...) + addend).  Segments with no stored source are skipped: adding
// their +0.0 changes no sum that started from 0.0.  This is what BlockMatrix.multiply(DistributedVector) computes with F2J
// dgemv per block column (segment) and the reduceByKey over the block row, because every term of a non-link is
// 0 * x_j = +0.0 for finite x_j >= 0.  A row's sum is one serial chain; it is never split into a tree.
//
// Rows are binned once, by in-degree:
//   degree <= MB_PAGERANK_LIGHT_BOUND  one lane per row.  A warp takes 32 consecutive rows, stages the contiguous edge span
//                                      of each run of light rows through shared memory with coalesced loads, and every
//                                      lane walks its own row there, gathering x through L2;
//   above                              one warp per row (the list made by pagerank_plan).  The lanes gather x and form the
//                                      products of the next chunk (each an exact single rounding) while lane 0 adds the
//                                      current chunk from shared memory, so the chain waits on DADD latency, not on
//                                      the gathers.
#include "pagerank.h"
#include "../../include/marlin_b200.h"
#include "launch.h"

#include <algorithm>

namespace mb {
namespace {

constexpr int LIGHT_BOUND = MB_PAGERANK_LIGHT_BOUND;
constexpr int ROW_WARPS = 4;          // warps per CTA of the light kernel
constexpr int STAGE = 512;            // edges a light warp stages per pass
constexpr int HEAVY_WARPS = 4;        // heavy rows per CTA
constexpr int DEPTH = 8;              // products per lane and chunk of a heavy row
constexpr int CHUNK = 32 * DEPTH;
constexpr unsigned FULL = 0xffffffffu;

// Adds p to the running partial acc of row state (tot, acc, end): a source j at or past the end of the current segment
// first folds acc into tot and starts the segment of j.
__device__ __forceinline__ void add_term(int j, double p, long long seg_len, double& tot, double& acc, long long& end) {
    if (j >= end) {
        tot = __dadd_rn(tot, acc);
        acc = 0.0;
        end = ((long long)j / seg_len + 1) * seg_len;
    }
    acc = __dadd_rn(acc, p);
}

__global__ void __launch_bounds__(256) pagerank_bin_kernel(CsrView L, int* heavy, int* count) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < L.rows; i += (long long)gridDim.x * blockDim.x)
        if (L.rowptr[i + 1] - L.rowptr[i] > LIGHT_BOUND) heavy[atomicAdd(count, 1)] = (int)i;
}

__global__ void __launch_bounds__(32 * ROW_WARPS) pagerank_step_kernel(CsrView L, const double* __restrict__ x,
                                                                       long long seg_len, double addend,
                                                                       double* __restrict__ y) {
    __shared__ int src_s[ROW_WARPS][STAGE];
    __shared__ double w_s[ROW_WARPS][STAGE];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const long long r0 = ((long long)blockIdx.x * ROW_WARPS + wid) * 32;
    if (r0 >= L.rows) return;                        // warp-uniform
    const long long i = r0 + lane;
    const bool valid = i < L.rows;
    const int a = valid ? L.rowptr[i] : 0, b = valid ? L.rowptr[i + 1] : 0;
    const bool light = valid && b - a <= LIGHT_BOUND;
    int* ss = src_s[wid];
    double* ws = w_s[wid];
    double tot = 0.0, acc = 0.0;
    long long end = -1;
    unsigned todo = __ballot_sync(FULL, light);
    while (todo) {
        // the run of consecutive light lanes [f, g): their edges are one contiguous span
        const int f = __ffs(todo) - 1;
        const unsigned gap = ~todo & (FULL << f);
        const int g = gap ? __ffs(gap) - 1 : 32;
        const int e0 = __shfl_sync(FULL, a, f), e1 = __shfl_sync(FULL, b, g - 1);
        const bool mine = lane >= f && lane < g;
        for (int c0 = e0; c0 < e1; c0 += STAGE) {
            const int cnt = min(STAGE, e1 - c0);
            for (int t = lane; t < cnt; t += 32) {
                ss[t] = L.colidx[c0 + t];
                ws[t] = L.vals[c0 + t];
            }
            __syncwarp();
            if (mine) {
                const int q1 = min(b, c0 + cnt);
                for (int q = max(a, c0) - c0; q < q1 - c0; ++q) {
                    const int j = ss[q];
                    add_term(j, __dmul_rn(ws[q], __ldg(x + j)), seg_len, tot, acc, end);
                }
            }
            __syncwarp();                            // the next pass overwrites the stage
        }
        todo = g == 32 ? 0u : todo & (FULL << g);
    }
    if (light) y[i] = __dadd_rn(__dadd_rn(tot, acc), addend);
}

__device__ __forceinline__ void heavy_load(const CsrView& L, long long c, long long b, int lane, int (&j)[DEPTH],
                                           double (&w)[DEPTH]) {
#pragma unroll
    for (int k = 0; k < DEPTH; ++k) {
        const long long q = c + k * 32 + lane;
        j[k] = q < b ? L.colidx[q] : -1;
        w[k] = q < b ? L.vals[q] : 0.0;
    }
}

__device__ __forceinline__ void heavy_gather(const double* __restrict__ x, const int (&j)[DEPTH], double (&v)[DEPTH]) {
#pragma unroll
    for (int k = 0; k < DEPTH; ++k) v[k] = j[k] >= 0 ? __ldg(x + j[k]) : 0.0;
}

// One warp per heavy row.  Chunk c's products and sources sit in shared memory while the lanes gather x for chunk c + 1
// and load the sources and weights of chunk c + 2; lane 0 then adds chunk c in order.
__global__ void __launch_bounds__(32 * HEAVY_WARPS) pagerank_step_kernel(CsrView L, const int* __restrict__ heavy, int nheavy,
                                                                         const double* __restrict__ x, long long seg_len,
                                                                         double addend, double* __restrict__ y) {
    __shared__ double prod_s[HEAVY_WARPS][CHUNK];
    __shared__ int src_s[HEAVY_WARPS][CHUNK];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const long long t = (long long)blockIdx.x * HEAVY_WARPS + wid;
    if (t >= nheavy) return;                         // warp-uniform
    const int i = heavy[t];
    const long long a = L.rowptr[i], b = L.rowptr[i + 1];
    double* ps = prod_s[wid];
    int* js = src_s[wid];
    int jc[DEPTH], jn[DEPTH];
    double wc[DEPTH], wn[DEPTH], xv[DEPTH];
    heavy_load(L, a, b, lane, jc, wc);
    heavy_gather(x, jc, xv);
    heavy_load(L, a + CHUNK, b, lane, jn, wn);
#pragma unroll
    for (int k = 0; k < DEPTH; ++k) {
        ps[k * 32 + lane] = __dmul_rn(wc[k], xv[k]);
        js[k * 32 + lane] = jc[k];
    }
    __syncwarp();
    double tot = 0.0, acc = 0.0;
    long long end = -1;
    for (long long c = a; c < b; c += CHUNK) {
        heavy_gather(x, jn, xv);
#pragma unroll
        for (int k = 0; k < DEPTH; ++k) {
            jc[k] = jn[k];
            wc[k] = wn[k];
        }
        heavy_load(L, c + 2 * CHUNK, b, lane, jn, wn);
        if (lane == 0) {
            const int cnt = (int)min((long long)CHUNK, b - c);
#pragma unroll 4
            for (int q = 0; q < cnt; ++q) add_term(js[q], ps[q], seg_len, tot, acc, end);
        }
        __syncwarp();
#pragma unroll
        for (int k = 0; k < DEPTH; ++k) {
            ps[k * 32 + lane] = __dmul_rn(wc[k], xv[k]);
            js[k * 32 + lane] = jc[k];
        }
        __syncwarp();
    }
    if (lane == 0) y[i] = __dadd_rn(__dadd_rn(tot, acc), addend);
}

}  // namespace

cudaError_t pagerank_plan(const CsrView& L, long long nnz, PagerankPlan* p, cudaStream_t st) {
    *p = PagerankPlan{};
    const long long cap = std::min<long long>(L.rows, nnz / (LIGHT_BOUND + 1));      // at most this many heavy rows
    cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&p->heavy), sizeof(int) * (size_t)(cap + 1));
    if (e != cudaSuccess) return e;
    int* count = p->heavy + cap;
    if ((e = cudaMemsetAsync(count, 0, sizeof(int), st)) != cudaSuccess) return e;
    if (cap > 0) {
        const unsigned grid = (unsigned)std::min<long long>((L.rows + 255) / 256, 4096);
        pagerank_bin_kernel<<<grid, 256, 0, st>>>(L, p->heavy, count);
        if ((e = launched()) != cudaSuccess) return e;
    }
    if ((e = cudaMemcpyAsync(&p->nheavy, count, sizeof(int), cudaMemcpyDeviceToHost, st)) != cudaSuccess) return e;
    return cudaStreamSynchronize(st);
}

cudaError_t pagerank_step(const CsrView& L, const PagerankPlan& p, const double* x, long long seg_len, double addend,
                          double* y, cudaStream_t st) {
    if (L.rows == 0) return cudaSuccess;
    const long long warps = (L.rows + 31) / 32;
    pagerank_step_kernel<<<(unsigned)((warps + ROW_WARPS - 1) / ROW_WARPS), 32 * ROW_WARPS, 0, st>>>(L, x, seg_len, addend, y);
    const cudaError_t e = launched();
    if (e != cudaSuccess || !p.nheavy) return e;
    pagerank_step_kernel<<<(unsigned)((p.nheavy + HEAVY_WARPS - 1) / HEAVY_WARPS), 32 * HEAVY_WARPS, 0, st>>>(
        L, p.heavy, p.nheavy, x, seg_len, addend, y);
    return launched();
}

}  // namespace mb

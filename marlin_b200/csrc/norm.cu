// DenseVecMatrix.norm (matrix/DenseVecMatrix.scala:975-999): the 1-, infinity- and Frobenius norms of an fp64 view, read
// once.
//
// norm_tile_kernel: every warp owns a sequence of 32 x 32 tiles and streams them through two shared-memory buffers with
// 8-byte cp.async copies, the next tile in flight while the current one is folded.  Consecutive lanes copy along the
// view's smaller stride (the columns of a row shard, the rows of a column-major block), so any view is read coalesced and
// in place.  The tiles of a warp come in tasks:
//   INF  a task is 32 rows, its tiles left to right; lane r folds row r in column order, s = s + |a| from 0.0, and the
//        warp keeps the largest row sum.
//   ONE  a task is one chunk of NORM_CHUNK rows and 32 columns, its tiles top to bottom; lane c sums column c over the
//        chunk in row order and writes the chunk partial.  norm_col_fold_kernel adds the partials in chunk order.
//   FRO  the tasks of ONE; each lane keeps Blue's three accumulators (LAPACK 3.10 dnrm2) over its column, the warp adds
//        the lanes' accumulators in a fixed tree and writes them per task; norm_fro_fold_kernel adds the tasks in a fixed
//        order.  Squares of entries above 2^486 or below 2^-511 are taken after scaling, so nothing overflows or underflows.
// The largest value is kept as the bits of a non-negative double (every sum here is one, or a positive NaN), whose
// unsigned order is java.lang.Double.compare's order, with atomicMax.  The task sizes do not depend on the grid, so every
// result is the same bits on every run.
#include "norm.h"
#include "launch.h"
#include "ptx.cuh"

#include <cstdint>

namespace mb {
namespace {

constexpr int NT = 32;                         // tile edge
constexpr int NP = NT + 1;                     // doubles per tile row in shared memory
constexpr int NORM_WARPS = 8;
constexpr int NORM_THREADS = NORM_WARPS * 32;
constexpr int NORM_CHUNK = 4096;               // rows per column-sum chunk
constexpr int NORM_SMEM = NORM_WARPS * 2 * NT * NP * 8;
constexpr int RESULT_DOUBLES = 4;              // head of the workspace: the results

// dnrm2's thresholds and scales for IEEE double (radix 2, minexponent -1021, maxexponent 1024, digits 53)
constexpr double TSML = 0x1p-511, TBIG = 0x1p486, SSML = 0x1p537, SBIG = 0x1p-538;

struct NormShape {
    const double* x;
    long long rs, cs;
    long long m;
    int n;
    int kind;
    int ncolt;                 // column tiles
    bool lane_is_col;          // lanes copy along the columns (cs <= rs)
    long long ntasks;
};

__device__ __forceinline__ void cp_async8(double* dst, const double* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ int tiles_in_task(const NormShape& s, long long task) {
    if (s.kind == NORM_INF) return s.ncolt;
    const long long rows = min((long long)NORM_CHUNK, s.m - (task / s.ncolt) * NORM_CHUNK);
    return static_cast<int>((rows + NT - 1) / NT);
}

__device__ __forceinline__ void tile_origin(const NormShape& s, long long task, int sub, long long* r0, int* c0) {
    if (s.kind == NORM_INF) {
        *r0 = task * NT;
        *c0 = sub * NT;
    } else {
        *r0 = (task / s.ncolt) * NORM_CHUNK + (long long)sub * NT;
        *c0 = static_cast<int>(task % s.ncolt) * NT;
    }
}

__device__ __forceinline__ void next_tile(const NormShape& s, long long* task, int* sub, long long stride) {
    if (++*sub == tiles_in_task(s, *task)) {
        *sub = 0;
        *task += stride;
    }
}

// The warp copies tile (task, sub) into `tile`; entries outside the view are 0.0.  Always commits one group.
__device__ __forceinline__ void issue_tile(const NormShape& s, long long task, int sub, double* tile, int lane) {
    if (task < s.ntasks) {
        long long r0;
        int c0;
        tile_origin(s, task, sub, &r0, &c0);
        const int nr = static_cast<int>(min((long long)NT, s.m - r0)), nc = min(NT, s.n - c0);
#pragma unroll 8
        for (int k = 0; k < NT; ++k) {
            const int i = s.lane_is_col ? k : lane, j = s.lane_is_col ? lane : k;
            double* d = tile + i * NP + j;
            if (i < nr && j < nc)
                cp_async8(d, s.x + (r0 + i) * s.rs + (long long)(c0 + j) * s.cs);
            else
                *d = 0.0;
        }
    }
    cp_async_commit();
}

__device__ __forceinline__ void blue_add(double ax, double& asml, double& amed, double& abig) {
    if (ax > TBIG) {
        const double y = __dmul_rn(ax, SBIG);
        abig = __dadd_rn(abig, __dmul_rn(y, y));
    } else if (ax < TSML) {
        const double y = __dmul_rn(ax, SSML);
        asml = __dadd_rn(asml, __dmul_rn(y, y));
    } else {
        amed = __dadd_rn(amed, __dmul_rn(ax, ax));          // NaN lands here
    }
}

__device__ __forceinline__ unsigned long long warp_max_bits(unsigned long long b) {
#pragma unroll
    for (int o = 16; o; o >>= 1) b = max(b, __shfl_xor_sync(0xffffffffu, b, o));
    return b;
}

__global__ void __launch_bounds__(NORM_THREADS, 1) norm_tile_kernel(NormShape s, double* part, unsigned long long* best_out) {
    extern __shared__ __align__(16) unsigned char norm_smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double* bufs = reinterpret_cast<double*>(norm_smem) + (size_t)warp * 2 * NT * NP;
    const long long stride = (long long)gridDim.x * NORM_WARPS;
    long long task = (long long)blockIdx.x * NORM_WARPS + warp, ptask = task;
    int sub = 0, psub = 0;
    issue_tile(s, ptask, psub, bufs, lane);
    if (ptask < s.ntasks) next_tile(s, &ptask, &psub, stride);
    double acc = 0.0, asml = 0.0, amed = 0.0, abig = 0.0;
    unsigned long long best = 0;                             // the bits of +0.0
    for (int k = 0; task < s.ntasks; ++k) {
        issue_tile(s, ptask, psub, bufs + ((k + 1) & 1) * NT * NP, lane);
        if (ptask < s.ntasks) next_tile(s, &ptask, &psub, stride);
        cp_async_wait<1>();
        __syncwarp();                                        // every lane's copies of tile k are visible
        const double* t = bufs + (k & 1) * NT * NP;
        if (sub == 0) acc = asml = amed = abig = 0.0;
        if (s.kind == NORM_INF) {
            const double* row = t + lane * NP;
#pragma unroll 8
            for (int j = 0; j < NT; ++j) acc = __dadd_rn(acc, fabs(row[j]));
        } else if (s.kind == NORM_ONE) {
#pragma unroll 8
            for (int i = 0; i < NT; ++i) acc = __dadd_rn(acc, fabs(t[i * NP + lane]));
        } else {
#pragma unroll 4
            for (int i = 0; i < NT; ++i) blue_add(fabs(t[i * NP + lane]), asml, amed, abig);
        }
        __syncwarp();                                        // the buffer is read before iteration k + 1 refills it
        if (sub == tiles_in_task(s, task) - 1) {
            long long r0;
            int c0;
            tile_origin(s, task, sub, &r0, &c0);
            if (s.kind == NORM_INF) {
                if (task * NT + lane < s.m) best = max(best, (unsigned long long)__double_as_longlong(acc));
            } else if (s.kind == NORM_ONE) {
                if (c0 + lane < s.n) part[(task / s.ncolt) * s.n + c0 + lane] = acc;
            } else {
#pragma unroll
                for (int o = 16; o; o >>= 1) {
                    asml = __dadd_rn(asml, __shfl_down_sync(0xffffffffu, asml, o));
                    amed = __dadd_rn(amed, __shfl_down_sync(0xffffffffu, amed, o));
                    abig = __dadd_rn(abig, __shfl_down_sync(0xffffffffu, abig, o));
                }
                if (lane == 0) {
                    part[task * 3 + 0] = asml;
                    part[task * 3 + 1] = amed;
                    part[task * 3 + 2] = abig;
                }
            }
        }
        next_tile(s, &task, &sub, stride);
    }
    cp_async_wait<0>();
    if (s.kind == NORM_INF) {
        best = warp_max_bits(best);
        if (lane == 0) atomicMax(best_out, best);
    }
}

// col[j * inc] = part[0][j] + part[1][j] + ... in chunk order; the largest column sum into *best_out
__global__ void __launch_bounds__(256) norm_col_fold_kernel(const double* part, long long nq, int n, double* col, long long inc,
                                                            unsigned long long* best_out) {
    const int j = blockIdx.x * 256 + threadIdx.x;
    unsigned long long b = 0;
    if (j < n) {
        double s = part[j];
#pragma unroll 16
        for (long long q = 1; q < nq; ++q) s = __dadd_rn(s, part[q * n + j]);
        col[j * inc] = s;
        b = (unsigned long long)__double_as_longlong(s);
    }
    b = warp_max_bits(b);
    if ((threadIdx.x & 31) == 0) atomicMax(best_out, b);
}

// out[0..2] = the per-task accumulators added up: thread t takes tasks t, t + 256, ... in order, then thread 0 adds the
// 256 thread sums in order
__global__ void __launch_bounds__(256) norm_fro_fold_kernel(const double* part, long long ntasks, double* out) {
    __shared__ double acc[3][256];
    double a0 = 0.0, a1 = 0.0, a2 = 0.0;
    for (long long t = threadIdx.x; t < ntasks; t += 256) {
        a0 = __dadd_rn(a0, part[t * 3 + 0]);
        a1 = __dadd_rn(a1, part[t * 3 + 1]);
        a2 = __dadd_rn(a2, part[t * 3 + 2]);
    }
    acc[0][threadIdx.x] = a0;
    acc[1][threadIdx.x] = a1;
    acc[2][threadIdx.x] = a2;
    __syncthreads();
    if (threadIdx.x < 3) {
        double s = 0.0;
        for (int i = 0; i < 256; ++i) s = __dadd_rn(s, acc[threadIdx.x][i]);
        out[threadIdx.x] = s;
    }
}

long long column_tiles(int n) { return (n + NT - 1) / NT; }
long long chunks(long long m) { return (m + NORM_CHUNK - 1) / NORM_CHUNK; }

}  // namespace

size_t norm_workspace_bytes(int kind, long long m, int n) {
    size_t part = 0;
    if (kind == NORM_ONE) part = (size_t)chunks(m) * (size_t)n;
    if (kind == NORM_FRO) part = (size_t)chunks(m) * (size_t)column_tiles(n) * 3;
    return (RESULT_DOUBLES + part) * sizeof(double);
}

cudaError_t norm_f64(int kind, const double* x, long long rs, long long cs, long long m, int n, double* col, long long inc,
                     void* ws, double** result, int num_sms, cudaStream_t st) {
    if (m <= 0 || n <= 0 || (kind != NORM_ONE && kind != NORM_INF && kind != NORM_FRO)) return cudaErrorInvalidValue;
    NormShape s;
    s.x = x;
    s.rs = rs;
    s.cs = cs;
    s.m = m;
    s.n = n;
    s.kind = kind;
    s.ncolt = static_cast<int>(column_tiles(n));
    s.lane_is_col = cs <= rs;
    s.ntasks = kind == NORM_INF ? (m + NT - 1) / NT : chunks(m) * s.ncolt;
    double* res = static_cast<double*>(ws);
    double* part = res + RESULT_DOUBLES;
    unsigned long long* best = reinterpret_cast<unsigned long long*>(res);
    cudaError_t e = cudaMemsetAsync(res, 0, RESULT_DOUBLES * sizeof(double), st);
    if (e != cudaSuccess) return e;
    const long long want = (s.ntasks + NORM_WARPS - 1) / NORM_WARPS;
    const int grid = static_cast<int>(want < num_sms ? want : num_sms);
    e = launch_with_smem<norm_tile_kernel>(grid, NORM_THREADS, NORM_SMEM, st, s, part, best);
    if (e != cudaSuccess) return e;
    if (kind == NORM_ONE) {
        norm_col_fold_kernel<<<(n + 255) / 256, 256, 0, st>>>(part, chunks(m), n, col, inc, best);
        e = launched();
    } else if (kind == NORM_FRO) {
        norm_fro_fold_kernel<<<1, 256, 0, st>>>(part, s.ntasks, res);
        e = launched();
    }
    if (e == cudaSuccess) *result = res;
    return e;
}

}  // namespace mb

// HBM-bound BLAS-2 / BLAS-1 block kernels of the vector side of the path: matrix x vector
// (SubMatrix.multiply(v: Vector), matrix/SubMatrix.scala:131-139 -> Breeze `BDM * BDV` -> netlib dgemv),
// vector . vector and vector x vector^T (DistributedVector.multiply, matrix/DistributedVector.scala:146-180
// -> Breeze `v.t * w` = ddot, `v * w.t` = rank-1 product).
//
// All three move each matrix element across HBM exactly once (gemv: 8*M*N bytes read, ger: 8*M*N written),
// one 16 KiB-ish tile of work per CTA like the element-wise kernels, and are deterministic: column chunks /
// row segments go to fixed CTAs, partial vectors are summed in ascending chunk order by a second launch.
// Multiplies and adds round separately (the JVM never contracts to an FMA), so a gemv that fits one column
// chunk reproduces F2J's dgemv bit for bit.
#include "blas12.h"
#include "launch.h"

#include <cstdint>

namespace mb {
namespace {

constexpr int GEMV_THREADS = 128;
constexpr int GEMV_ROWS = GEMV_THREADS * 2;      // rows per CTA in the N kernel (one double2 per thread)
constexpr int GEMV_MAX_CHUNK = 512;              // columns per CTA (x chunk staged in shared memory)
constexpr int GEMV_T_WARPS = 8;
constexpr int GEMV_T_SEG = 2048;                 // rows per (warp, segment) in the T kernel: 16 KiB of one column

// ---- y = A x, A column-major m x n (lda).  grid (ceil(m/256), chunks).  part[chunk*m + r] ----
__global__ void __launch_bounds__(GEMV_THREADS) gemv_n_kernel(const double* a, long long lda, int m, int n,
                                                              const double* x, long long incx, double* part, int cb) {
    __shared__ double xs[GEMV_MAX_CHUNK];
    const int c0 = blockIdx.y * cb;
    const int nc = min(cb, n - c0);
    for (int i = threadIdx.x; i < nc; i += GEMV_THREADS) xs[i] = x[(long long)(c0 + i) * incx];
    __syncthreads();
    const int r = (blockIdx.x * GEMV_THREADS + threadIdx.x) * 2;
    if (r >= m) return;
    const double* col = a + (long long)c0 * lda + r;
    double* out = part + (long long)blockIdx.y * m + r;
    const bool vec = (r + 1 < m) && ((lda & 1) == 0) && ((reinterpret_cast<uintptr_t>(a) & 15) == 0);
    if (vec) {
        double y0 = 0.0, y1 = 0.0;
        int c = 0;
        for (; c + 8 <= nc; c += 8) {
            double2 v[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) v[u] = *reinterpret_cast<const double2*>(col + (long long)(c + u) * lda);
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const double t = xs[c + u];
                if (t == 0.0) continue;            // dgemv 'N' skips x(j) = 0: an Inf / NaN in that column is not read
                y0 = __dadd_rn(y0, __dmul_rn(t, v[u].x));
                y1 = __dadd_rn(y1, __dmul_rn(t, v[u].y));
            }
        }
        for (; c < nc; ++c) {
            const double2 v = *reinterpret_cast<const double2*>(col + (long long)c * lda);
            const double t = xs[c];
            if (t == 0.0) continue;
            y0 = __dadd_rn(y0, __dmul_rn(t, v.x));
            y1 = __dadd_rn(y1, __dmul_rn(t, v.y));
        }
        out[0] = y0;
        out[1] = y1;
    } else {
        const int nr = min(2, m - r);
        for (int q = 0; q < nr; ++q) {
            double y = 0.0;
            int c = 0;
            for (; c + 4 <= nc; c += 4) {
                double v[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) v[u] = col[(long long)(c + u) * lda + q];
#pragma unroll
                for (int u = 0; u < 4; ++u)
                    if (xs[c + u] != 0.0) y = __dadd_rn(y, __dmul_rn(xs[c + u], v[u]));
            }
            for (; c < nc; ++c)
                if (xs[c] != 0.0) y = __dadd_rn(y, __dmul_rn(xs[c], col[(long long)c * lda + q]));
            out[q] = y;
        }
    }
}

// ---- y = A^T x, A column-major m x n (lda): one warp per (column, row segment); part[seg*n + col] ----
__global__ void __launch_bounds__(GEMV_T_WARPS * 32) gemv_t_kernel(const double* a, long long lda, int m, int n,
                                                                   const double* x, long long incx, double* part) {
    const int col = blockIdx.x * GEMV_T_WARPS + (threadIdx.x >> 5);
    if (col >= n) return;
    const int lane = threadIdx.x & 31;
    const int r0 = blockIdx.y * GEMV_T_SEG;
    const int nr = min(GEMV_T_SEG, m - r0);
    const double* p = a + (long long)col * lda + r0;
    const double* xv = x + (long long)r0 * incx;
    double s0 = 0.0, s1 = 0.0;
    const bool vec = incx == 1 && ((lda & 1) == 0) && ((reinterpret_cast<uintptr_t>(a) & 15) == 0) &&
                     ((reinterpret_cast<uintptr_t>(x) & 15) == 0) && ((r0 & 1) == 0);
    int done = 0;
    if (vec) {
        const int pairs = nr >> 1;
        int i = lane;
        for (; i + 96 < pairs; i += 128) {
            double2 av[4], xw[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                av[u] = reinterpret_cast<const double2*>(p)[i + 32 * u];
                xw[u] = reinterpret_cast<const double2*>(xv)[i + 32 * u];
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                s0 = __dadd_rn(s0, __dmul_rn(av[u].x, xw[u].x));
                s1 = __dadd_rn(s1, __dmul_rn(av[u].y, xw[u].y));
            }
        }
        for (; i < pairs; i += 32) {
            const double2 av = reinterpret_cast<const double2*>(p)[i];
            const double2 xw = reinterpret_cast<const double2*>(xv)[i];
            s0 = __dadd_rn(s0, __dmul_rn(av.x, xw.x));
            s1 = __dadd_rn(s1, __dmul_rn(av.y, xw.y));
        }
        done = pairs * 2;
    }
    for (int i = done + lane; i < nr; i += 32) s0 = __dadd_rn(s0, __dmul_rn(p[i], xv[(long long)i * incx]));
    double s = __dadd_rn(s0, s1);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s = __dadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
    if (lane == 0) part[(long long)blockIdx.y * n + col] = s;
}

// y[i] = (accumulate ? y[i] : 0) + part[0][i] + part[1][i] + ...  (ascending, fixed order)
__global__ void __launch_bounds__(256) fold_partials_kernel(const double* part, int nparts, int len, double* y,
                                                            long long incy, int accumulate) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= len) return;
    double s = nparts > 0 ? part[i] : 0.0;
    int p = 1;
    for (; p + 8 <= nparts; p += 8) {            // loads in flight together, adds in ascending order
        double v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) v[u] = part[(long long)(p + u) * len + i];
#pragma unroll
        for (int u = 0; u < 8; ++u) s = __dadd_rn(s, v[u]);
    }
    for (; p < nparts; ++p) s = __dadd_rn(s, part[(long long)p * len + i]);
    double* o = y + (long long)i * incy;
    *o = accumulate ? __dadd_rn(*o, s) : s;
}

// ---- out = x y^T (column-major m x n, ldo); 256 rows x 8 columns per CTA ----
constexpr int GER_COLS = 8;
__global__ void __launch_bounds__(GEMV_THREADS) ger_kernel(int m, int n, const double* x, long long incx, const double* y,
                                                           long long incy, double* out, long long ldo) {
    const int r = (blockIdx.y * GEMV_THREADS + threadIdx.x) * 2;
    if (r >= m) return;
    const int c0 = blockIdx.x * GER_COLS;
    const int nc = min(GER_COLS, n - c0);
    const double x0 = x[(long long)r * incx];
    const double x1 = (r + 1 < m) ? x[(long long)(r + 1) * incx] : 0.0;
    double* o = out + (long long)c0 * ldo + r;
    const bool vec = (r + 1 < m) && ((ldo & 1) == 0) && ((reinterpret_cast<uintptr_t>(out) & 15) == 0);
    // dgemm with k = 1 and beta = 0 computes 0 + y_j * x_i: the leading zero turns a -0.0 product into +0.0
#pragma unroll
    for (int c = 0; c < GER_COLS; ++c) {
        if (c < nc) {
            const double t = y[(long long)(c0 + c) * incy];
            const double v0 = __dadd_rn(0.0, __dmul_rn(t, x0)), v1 = __dadd_rn(0.0, __dmul_rn(t, x1));
            if (vec) {
                *reinterpret_cast<double2*>(o + (long long)c * ldo) = make_double2(v0, v1);
            } else {
                o[(long long)c * ldo] = v0;
                if (r + 1 < m) o[(long long)c * ldo + 1] = v1;
            }
        }
    }
}

// ---- dot: stage 1, one 2048-element tile per CTA; stage 2 folds the CTA partials in order ----
constexpr int DOT_TILE = 2048;
__device__ __forceinline__ double cta_reduce(double v) {
    __shared__ double sh[8];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x < 32) {
        t = threadIdx.x < 8 ? sh[threadIdx.x] : 0.0;
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) t = __dadd_rn(t, __shfl_xor_sync(0xffffffffu, t, o));
    }
    return t;
}

__global__ void __launch_bounds__(256) dot_stage1_kernel(long long n, const double* x, long long incx, const double* y,
                                                         long long incy, double* part, int nparts) {
    double s = 0.0;
    const long long tiles = (n + DOT_TILE - 1) / DOT_TILE;
    const bool vec = incx == 1 && incy == 1 && ((reinterpret_cast<uintptr_t>(x) & 15) == 0) &&
                     ((reinterpret_cast<uintptr_t>(y) & 15) == 0);
    for (long long t = blockIdx.x; t < tiles; t += nparts) {
        const long long base = t * DOT_TILE;
        if (vec && base + DOT_TILE <= n) {
            double2 a[4], b[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                a[u] = reinterpret_cast<const double2*>(x + base)[threadIdx.x + 256 * u];
                b[u] = reinterpret_cast<const double2*>(y + base)[threadIdx.x + 256 * u];
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) s = __dadd_rn(s, __dadd_rn(__dmul_rn(a[u].x, b[u].x), __dmul_rn(a[u].y, b[u].y)));
        } else {
            for (long long i = base + threadIdx.x; i < min(n, base + DOT_TILE); i += 256)
                s = __dadd_rn(s, __dmul_rn(x[i * incx], y[i * incy]));
        }
    }
    const double t = cta_reduce(s);
    if (threadIdx.x == 0) part[blockIdx.x] = t;
}

__global__ void __launch_bounds__(256) dot_stage2_kernel(const double* part, int n, double* out) {
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += 256) s = __dadd_rn(s, part[i]);
    const double t = cta_reduce(s);
    if (threadIdx.x == 0) *out = t;
}

}  // namespace

int gemv_chunk_cols(int n) {
    // 256 columns per CTA (128 x 2 rows x 256 columns = 512 KiB of A per CTA); 512 once that would make more than
    // 64 partial vectors
    int cb = 256;
    if ((n + cb - 1) / cb > 64) cb = GEMV_MAX_CHUNK;
    return cb;
}

size_t gemv_workspace_doubles(bool trans, int m, int n) {
    if (!trans) {
        const int cb = gemv_chunk_cols(n);
        const long long chunks = (n + cb - 1) / cb;
        return (size_t)(chunks > 0 ? chunks : 1) * (size_t)(m > 0 ? m : 1);
    }
    const long long segs = (m + GEMV_T_SEG - 1) / GEMV_T_SEG;
    return (size_t)(segs > 0 ? segs : 1) * (size_t)(n > 0 ? n : 1);
}

cudaError_t gemv_f64(bool trans, int m, int n, const double* a, long long lda, const double* x, long long incx, double* y,
                     long long incy, bool accumulate, double* workspace, cudaStream_t st) {
    const int len = trans ? n : m;          // result length
    const int red = trans ? m : n;          // contraction length
    if (len == 0) return cudaSuccess;
    if (red == 0) {
        // empty contraction: y = 0 (or unchanged when accumulating), like dgemv with beta = 0 / 1
        if (accumulate) return cudaSuccess;
        fold_partials_kernel<<<(len + 255) / 256, 256, 0, st>>>(workspace, 0, len, y, incy, 0);
        return launched();
    }
    int nparts;
    if (!trans) {
        const int cb = gemv_chunk_cols(n);
        nparts = (n + cb - 1) / cb;
        if (nparts > 65535) return cudaErrorInvalidValue;
        dim3 grid((m + GEMV_ROWS - 1) / GEMV_ROWS, nparts);
        gemv_n_kernel<<<grid, GEMV_THREADS, 0, st>>>(a, lda, m, n, x, incx, workspace, cb);
    } else {
        nparts = (m + GEMV_T_SEG - 1) / GEMV_T_SEG;
        if (nparts > 65535) return cudaErrorInvalidValue;
        dim3 grid((n + GEMV_T_WARPS - 1) / GEMV_T_WARPS, nparts);
        gemv_t_kernel<<<grid, GEMV_T_WARPS * 32, 0, st>>>(a, lda, m, n, x, incx, workspace);
    }
    if (const cudaError_t e = launched(); e != cudaSuccess) return e;
    fold_partials_kernel<<<(len + 255) / 256, 256, 0, st>>>(workspace, nparts, len, y, incy, accumulate ? 1 : 0);
    return launched();
}

cudaError_t ger_f64(int m, int n, const double* x, long long incx, const double* y, long long incy, double* out,
                    long long ldo, cudaStream_t st) {
    if (m == 0 || n == 0) return cudaSuccess;
    dim3 grid((n + GER_COLS - 1) / GER_COLS, (m + GEMV_ROWS - 1) / GEMV_ROWS);
    if (grid.y > 65535) return cudaErrorInvalidValue;
    ger_kernel<<<grid, GEMV_THREADS, 0, st>>>(m, n, x, incx, y, incy, out, ldo);
    return launched();
}

int dot_scratch_doubles() { return 4096 + 1; }

cudaError_t dot_f64(long long n, const double* x, long long incx, const double* y, long long incy, double* scratch,
                    cudaStream_t st) {
    const long long tiles = (n + DOT_TILE - 1) / DOT_TILE;
    const int nparts = (int)(tiles < 1 ? 1 : (tiles > 4096 ? 4096 : tiles));
    dot_stage1_kernel<<<nparts, 256, 0, st>>>(n, x, incx, y, incy, scratch + 1, nparts);
    if (const cudaError_t e = launched(); e != cudaSuccess) return e;
    dot_stage2_kernel<<<1, 256, 0, st>>>(scratch + 1, nparts, scratch);
    return launched();
}

}  // namespace mb

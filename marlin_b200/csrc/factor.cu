// Dense factorizations of one device block — the local step of DenseVecMatrix.luDecompose / choleskyDecompose / inverse
// (matrix/DenseVecMatrix.scala:283-466, 475-561, 568-764), which the reference delegates to Breeze -> LAPACK
// (`brzLU` = dgetrf, `brzCholesky` = dpotrf, `brzInv` = dgetrf + dgetri, `\` = dgesv / dtrtrs).
//
// Everything is recursive (Toledo-style): a factorization of n columns splits into two halves joined by a triangular
// solve and a rank-n/2 update, so ~all flops land in the DMMA GEMM (gemm_f64.cu) and only the leaves run here:
//   * lu_panel_kernel      — partial-pivoting LU of a tall (rows x <=32) panel, one CTA, LAPACK dgetf2 conventions
//                            (first maximal |a| wins, reciprocal scaling);
//   * laswp_kernel         — row interchanges on a column range;
//   * trsm_leaf_kernel     — T X = B for a <=64 x 64 triangle staged in shared memory, one right-hand side per thread;
//   * potrf_leaf_kernel    — Cholesky of a <=64 x 64 block in shared memory.
// All kernels take element strides (rs, cs), so Breeze views (transposed, sliced) need no copies.
#include "factor.h"
#include "gemm_f64.h"
#include "launch.h"

#include <algorithm>
#include <cfloat>

namespace mb {

namespace {

constexpr int PANEL_W = 32;
constexpr int LEAF = 64;

__global__ void __launch_bounds__(1024)
lu_panel_kernel(double* a, long long rs, long long cs, int rows, int w, int* piv, int row_base, int* info) {
    __shared__ double s_val[32];
    __shared__ int s_idx[32];
    __shared__ double s_row[PANEL_W];
    __shared__ int s_p;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int steps = min(w, rows);
    for (int c = 0; c < steps; ++c) {
        // 1. pivot: first row with the largest |a[r][c]|, r >= c   (idamax)
        double best = -1.0;
        int bi = c;
        for (int r = c + tid; r < rows; r += 1024) {
            const double v = fabs(a[r * rs + c * cs]);
            if (v > best) { best = v; bi = r; }
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            const double ov = __shfl_down_sync(0xffffffffu, best, off);
            const int oi = __shfl_down_sync(0xffffffffu, bi, off);
            if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
        }
        if (lane == 0) { s_val[warp] = best; s_idx[warp] = bi; }
        __syncthreads();
        if (warp == 0) {
            best = s_val[lane];
            bi = s_idx[lane];
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) {
                const double ov = __shfl_down_sync(0xffffffffu, best, off);
                const int oi = __shfl_down_sync(0xffffffffu, bi, off);
                if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
            }
            if (lane == 0) {
                s_p = bi;
                piv[c] = row_base + bi;
                if (best == 0.0 && info && *info == 0) *info = row_base + c + 1;      // exactly singular (dgetf2's INFO)
            }
        }
        __syncthreads();
        const int p = s_p;
        // 2. interchange rows c and p inside the panel
        if (p != c && tid < w) {
            const double t = a[c * rs + tid * cs];
            a[c * rs + tid * cs] = a[p * rs + tid * cs];
            a[p * rs + tid * cs] = t;
        }
        __syncthreads();
        if (tid < w) s_row[tid] = a[c * rs + tid * cs];
        __syncthreads();
        const double pv = s_row[c];
        if (pv != 0.0) {
            // 3. + 4. scale the column by the reciprocal (dgetf2) and update the rest of the panel; like dgetf2, divide
            // instead when |pv| < sfmin = DBL_MIN, whose reciprocal overflows (1 / 2^-1060 = +Inf)
            const bool recip = fabs(pv) >= DBL_MIN;
            const double rinv = 1.0 / pv;
            for (int r = c + 1 + tid; r < rows; r += 1024) {
                const double l = recip ? a[r * rs + c * cs] * rinv : a[r * rs + c * cs] / pv;
                a[r * rs + c * cs] = l;
                for (int cc = c + 1; cc < w; ++cc) a[r * rs + cc * cs] -= l * s_row[cc];
            }
        }
        __syncthreads();
    }
}

// rows k0..k1-1: swap row k with row piv[k] (absolute indices) on columns [0, cols) of the view
__global__ void laswp_kernel(double* a, long long rs, long long cs, int cols, const int* piv, int k0, int k1) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= cols) return;
    double* col = a + (long long)c * cs;
    for (int k = k0; k < k1; ++k) {
        const int p = piv[k];
        if (p != k) {
            const double t = col[k * rs];
            col[k * rs] = col[p * rs];
            col[p * rs] = t;
        }
    }
}

// T X = B, T (t x t, t <= 64) lower or upper triangular, B (t x nrhs) overwritten by X.  One right-hand side per thread.
template <bool LOWER, bool UNIT>
__global__ void __launch_bounds__(128)
trsm_leaf_kernel(const double* T, long long trs, long long tcs, int t, double* B, long long brs, long long bcs, int nrhs) {
    __shared__ double sT[LEAF][LEAF + 1];
    for (int e = threadIdx.x; e < t * t; e += blockDim.x) {
        const int i = e % t, j = e / t;
        sT[i][j] = T[i * trs + j * tcs];
    }
    __syncthreads();
    const int col = blockIdx.x * blockDim.x + threadIdx.x;
    if (col >= nrhs) return;
    double x[LEAF];
    double* b = B + (long long)col * bcs;
    for (int i = 0; i < t; ++i) x[i] = b[i * brs];
    if (LOWER) {
        for (int i = 0; i < t; ++i) {
            double s = x[i];
            for (int j = 0; j < i; ++j) s -= sT[i][j] * x[j];
            x[i] = UNIT ? s : s / sT[i][i];
        }
    } else {
        for (int i = t - 1; i >= 0; --i) {
            double s = x[i];
            for (int j = i + 1; j < t; ++j) s -= sT[i][j] * x[j];
            x[i] = UNIT ? s : s / sT[i][i];
        }
    }
    for (int i = 0; i < t; ++i) b[i * brs] = x[i];
}

// Cholesky (lower) of a t x t block, t <= 64, in shared memory; only the lower triangle is read and written.
__global__ void __launch_bounds__(256)
potrf_leaf_kernel(double* a, long long rs, long long cs, int t, int row_base, int* info) {
    __shared__ double s[LEAF][LEAF + 1];
    __shared__ int bad;
    for (int e = threadIdx.x; e < t * t; e += blockDim.x) {
        const int i = e % t, j = e / t;
        if (i >= j) s[i][j] = a[i * rs + j * cs];
    }
    if (threadIdx.x == 0) bad = 0;
    __syncthreads();
    for (int j = 0; j < t; ++j) {
        if (threadIdx.x == 0) {
            double d = s[j][j];
            for (int p = 0; p < j; ++p) d -= s[j][p] * s[j][p];
            if (!(d > 0.0)) { bad = j + 1; d = 1.0; }
            s[j][j] = sqrt(d);
        }
        __syncthreads();
        const double djj = s[j][j];
        for (int i = j + 1 + threadIdx.x; i < t; i += blockDim.x) {
            double v = s[i][j];
            for (int p = 0; p < j; ++p) v -= s[i][p] * s[j][p];
            s[i][j] = v / djj;
        }
        __syncthreads();
    }
    for (int e = threadIdx.x; e < t * t; e += blockDim.x) {
        const int i = e % t, j = e / t;
        if (i >= j) a[i * rs + j * cs] = s[i][j];
    }
    if (threadIdx.x == 0 && bad && info && *info == 0) *info = row_base + bad;   // not positive definite (dpotrf's INFO)
}

__global__ void zero_strict_upper_kernel(double* a, long long rs, long long cs, int n) {
    const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (e >= (long long)n * n) return;
    const int i = (int)(e % n), j = (int)(e / n);
    if (i < j) a[i * rs + j * cs] = 0.0;
}

// out (n x n) = rows of the identity permuted: out[i][perm_row(i)] ... built as I, the caller applies laswp
__global__ void identity_kernel(double* a, long long rs, long long cs, int n) {
    const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (e >= (long long)n * n) return;
    const int i = (int)(e % n), j = (int)(e / n);
    a[i * rs + j * cs] = (i == j) ? 1.0 : 0.0;
}

// ipiv (swap sequence, absolute rows) -> permutation array: row i of P*A is row perm[i] of A (the reference's pArray)
__global__ void ipiv_to_perm_kernel(const int* piv, int n, int* perm) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    for (int i = 0; i < n; ++i) perm[i] = i;
    for (int i = 0; i < n; ++i) {
        const int p = piv[i];
        const int t = perm[i];
        perm[i] = perm[p];
        perm[p] = t;
    }
}

inline int split(int n) {
    // first half: a multiple of 32 close to n / 2
    int h = ((n / 2 + 31) / 32) * 32;
    if (h >= n) h = (n / 2 / 32) * 32;
    if (h <= 0) h = n / 2;
    return h;
}

// C (view) = alpha * A * B + beta * C with arbitrary element strides on all three: routed to the column-major GEMM
cudaError_t gemm_view(const FView& A, const FView& B, const FView& C, double alpha, double beta, int num_sms, cudaStream_t st) {
    // a view is "N" when rs == 1 (column-major, ld = cs) and "T" when cs == 1 (row-major, ld = rs)
    auto form = [](const FView& v, bool* trans, long long* ld) {
        if (v.rs == 1) { *trans = false; *ld = v.cs; return true; }
        if (v.cs == 1) { *trans = true; *ld = v.rs; return true; }
        return false;
    };
    bool ta, tb, tc;
    long long lda, ldb, ldc;
    if (!form(A, &ta, &lda) || !form(B, &tb, &ldb) || !form(C, &tc, &ldc)) return cudaErrorInvalidValue;
    if (lda < 1) lda = 1;
    if (ldb < 1) ldb = 1;
    if (ldc < 1) ldc = 1;
    const int M = C.rows, N = C.cols, K = A.cols;
    if (!tc) return gemm_f64(ta, tb, M, N, K, alpha, A.p, lda, B.p, ldb, beta, C.p, ldc, num_sms, st, false);
    // C^T = B^T * A^T on the column-major array underneath
    return gemm_f64(!tb, !ta, N, M, K, alpha, B.p, ldb, A.p, lda, beta, C.p, ldc, num_sms, st, false);
}

inline FView sub(const FView& v, int r0, int r1, int c0, int c1) {
    return FView{v.p + r0 * v.rs + c0 * v.cs, v.rs, v.cs, r1 - r0, c1 - c0};
}
inline FView tr(const FView& v) { return FView{v.p, v.cs, v.rs, v.cols, v.rows}; }

}  // namespace

// ---- T X = B (left side), T triangular t x t, B t x nrhs, in place -------------------------------------------------
cudaError_t trsm_left(const FView& T, bool lower, bool unit, const FView& B, int num_sms, cudaStream_t st) {
    const int t = T.rows, nrhs = B.cols;
    if (t <= 0 || nrhs <= 0) return cudaSuccess;
    if (t <= LEAF) {
        const int blocks = (nrhs + 127) / 128;
        if (lower && unit) trsm_leaf_kernel<true, true><<<blocks, 128, 0, st>>>(T.p, T.rs, T.cs, t, B.p, B.rs, B.cs, nrhs);
        else if (lower) trsm_leaf_kernel<true, false><<<blocks, 128, 0, st>>>(T.p, T.rs, T.cs, t, B.p, B.rs, B.cs, nrhs);
        else if (unit) trsm_leaf_kernel<false, true><<<blocks, 128, 0, st>>>(T.p, T.rs, T.cs, t, B.p, B.rs, B.cs, nrhs);
        else trsm_leaf_kernel<false, false><<<blocks, 128, 0, st>>>(T.p, T.rs, T.cs, t, B.p, B.rs, B.cs, nrhs);
        return launched();
    }
    const int h = split(t);
    const FView T11 = sub(T, 0, h, 0, h), T22 = sub(T, h, t, h, t);
    const FView B1 = sub(B, 0, h, 0, nrhs), B2 = sub(B, h, t, 0, nrhs);
    cudaError_t e;
    if (lower) {
        if ((e = trsm_left(T11, true, unit, B1, num_sms, st)) != cudaSuccess) return e;
        if ((e = gemm_view(sub(T, h, t, 0, h), B1, B2, -1.0, 1.0, num_sms, st)) != cudaSuccess) return e;
        return trsm_left(T22, true, unit, B2, num_sms, st);
    }
    if ((e = trsm_left(T22, false, unit, B2, num_sms, st)) != cudaSuccess) return e;
    if ((e = gemm_view(sub(T, 0, h, h, t), B2, B1, -1.0, 1.0, num_sms, st)) != cudaSuccess) return e;
    return trsm_left(T11, false, unit, B1, num_sms, st);
}

namespace {

// LU of the (m x n) view `a` = columns [c0, c0+n) / rows [r0, ...) of the full matrix `full`; pivots are absolute rows.
cudaError_t getrf_rec(const FView& full, int r0, int c0, int m, int n, int* piv, int* info, int num_sms, cudaStream_t st) {
    if (m <= 0 || n <= 0) return cudaSuccess;
    const FView a = sub(full, r0, r0 + m, c0, c0 + n);
    if (n <= PANEL_W) {
        lu_panel_kernel<<<1, 1024, 0, st>>>(a.p, a.rs, a.cs, m, n, piv + r0, r0, info);
        return launched();
    }
    const int n1 = std::min(split(n), m);
    const int n2 = n - n1;
    cudaError_t e;
    if ((e = getrf_rec(full, r0, c0, m, n1, piv, info, num_sms, st)) != cudaSuccess) return e;
    const int k1 = std::min(m, n1);
    // apply the left half's interchanges to the right half
    const FView right_full = sub(full, 0, full.rows, c0 + n1, c0 + n);
    laswp_kernel<<<(n2 + 127) / 128, 128, 0, st>>>(right_full.p, right_full.rs, right_full.cs, n2, piv, r0, r0 + k1);
    if ((e = launched()) != cudaSuccess) return e;
    // U12 = L11^-1 A12;  A22 -= L21 U12
    const FView L11 = sub(full, r0, r0 + k1, c0, c0 + k1);
    const FView A12 = sub(full, r0, r0 + k1, c0 + n1, c0 + n);
    if ((e = trsm_left(L11, true, true, A12, num_sms, st)) != cudaSuccess) return e;
    if (m > k1) {
        const FView L21 = sub(full, r0 + k1, r0 + m, c0, c0 + k1);
        const FView A22 = sub(full, r0 + k1, r0 + m, c0 + n1, c0 + n);
        if ((e = gemm_view(L21, A12, A22, -1.0, 1.0, num_sms, st)) != cudaSuccess) return e;
        if ((e = getrf_rec(full, r0 + k1, c0 + n1, m - k1, n2, piv, info, num_sms, st)) != cudaSuccess) return e;
        // the right half's interchanges, applied back to the left half
        const int k2 = std::min(m - k1, n2);
        const FView left_full = sub(full, 0, full.rows, c0, c0 + n1);
        laswp_kernel<<<(n1 + 127) / 128, 128, 0, st>>>(left_full.p, left_full.rs, left_full.cs, n1, piv, r0 + k1, r0 + k1 + k2);
        if ((e = launched()) != cudaSuccess) return e;
    }
    return cudaSuccess;
}

cudaError_t potrf_rec(const FView& full, int r0, int n, int* info, int num_sms, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    if (n <= LEAF) {
        const FView a = sub(full, r0, r0 + n, r0, r0 + n);
        potrf_leaf_kernel<<<1, 256, 0, st>>>(a.p, a.rs, a.cs, n, r0, info);
        return launched();
    }
    const int n1 = split(n), n2 = n - n1;
    cudaError_t e;
    if ((e = potrf_rec(full, r0, n1, info, num_sms, st)) != cudaSuccess) return e;
    const FView L11 = sub(full, r0, r0 + n1, r0, r0 + n1);
    const FView A21 = sub(full, r0 + n1, r0 + n, r0, r0 + n1);
    // X L11^T = A21  <=>  L11 X^T = A21^T
    if ((e = trsm_left(L11, true, false, tr(A21), num_sms, st)) != cudaSuccess) return e;
    const FView A22 = sub(full, r0 + n1, r0 + n, r0 + n1, r0 + n);
    if ((e = gemm_view(A21, tr(A21), A22, -1.0, 1.0, num_sms, st)) != cudaSuccess) return e;
    (void)n2;
    return potrf_rec(full, r0 + n1, n - n1, info, num_sms, st);
}

}  // namespace

cudaError_t getrf(const FView& a, int* piv_dev, int* perm_dev, int* info_dev, int num_sms, cudaStream_t st) {
    const int k = std::min(a.rows, a.cols);
    cudaError_t e = cudaMemsetAsync(info_dev, 0, sizeof(int), st);
    if (e != cudaSuccess) return e;
    if ((e = getrf_rec(a, 0, 0, a.rows, a.cols, piv_dev, info_dev, num_sms, st)) != cudaSuccess) return e;
    if (perm_dev) {
        // rows beyond min(m, n) are never pivot positions: identity there
        ipiv_to_perm_kernel<<<1, 1, 0, st>>>(piv_dev, k, perm_dev);
        e = launched();
    }
    return e;
}

cudaError_t potrf_lower(const FView& a, int* info_dev, int num_sms, cudaStream_t st) {
    cudaError_t e = cudaMemsetAsync(info_dev, 0, sizeof(int), st);
    if (e != cudaSuccess) return e;
    if ((e = potrf_rec(a, 0, a.rows, info_dev, num_sms, st)) != cudaSuccess) return e;
    const long long total = (long long)a.rows * a.rows;
    zero_strict_upper_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(a.p, a.rs, a.cs, a.rows);
    return launched();
}

// out = a^-1 : LU of a working copy `lu` (caller-provided, holds a on entry), then L (U X) = P I
cudaError_t inverse_from_lu(const FView& lu, const int* piv_dev, const FView& out, int num_sms, cudaStream_t st) {
    const int n = lu.rows;
    const long long total = (long long)n * n;
    identity_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(out.p, out.rs, out.cs, n);
    cudaError_t e = launched();
    if (e != cudaSuccess) return e;
    laswp_kernel<<<(n + 127) / 128, 128, 0, st>>>(out.p, out.rs, out.cs, n, piv_dev, 0, n);
    if ((e = launched()) != cudaSuccess) return e;
    if ((e = trsm_left(lu, true, true, out, num_sms, st)) != cudaSuccess) return e;
    return trsm_left(lu, false, false, out, num_sms, st);
}

}  // namespace mb

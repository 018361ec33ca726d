// Sparse (CSC) blocks: toDense, the three products of SubMatrix.multiply with a sparse side (matrix/SubMatrix.scala:87-119)
// and the row sampling of the sparse generator.
//
// Every output element is summed by one thread (or one warp lane) in the order of the reference's loop, with separate
// round-to-nearest multiplies and adds (__dmul_rn / __dadd_rn, never a fused multiply-add: the JVM does not fuse), starting
// from 0.0.  No value is ever combined with an atomic, so results are bitwise reproducible and bit-identical to a plain
// restatement of the reference loops.  `accumulate` adds the finished product to C once: D = C + P, the reduceByKey(add)
// of BlockMatrix.multiply (matrix/BlockMatrix.scala:177).
#include "sparse.h"
#include "elementwise.h"
#include "launch.h"
#include "stream_buffer.h"

#include <algorithm>

namespace mb {
namespace {

__device__ __forceinline__ double put(const double* o, double v, int accumulate) {
    return accumulate ? __dadd_rn(*o, v) : v;
}

// Matrices.scala:106-119: zeros, then each stored value in place.  One CTA per column; the barrier orders the two writes.
__global__ void __launch_bounds__(256) csc_to_dense_kernel(CscView S, DView out) {
    const int j = blockIdx.x;
    double* col = out.p + (long long)j * out.cs;
    for (int r = threadIdx.x; r < S.rows; r += blockDim.x) col[(long long)r * out.rs] = 0.0;
    __syncthreads();
    const int p1 = S.colptr[j + 1];
    for (int p = S.colptr[j] + threadIdx.x; p < p1; p += blockDim.x) col[(long long)S.rowidx[p] * out.rs] = S.vals[p];
}

// LibMatrixMult.multDenseSparse (LibMatrixMult.scala:15-41): C(:, j) = sum over the stored k of B(:, j), in stored order, of
// B(k, j) * A(:, k).  A column of B holding exactly one value equal to 1.0 is a copy of the A column (:28-29), which keeps
// -0.0.  Column j = blockIdx.x; consecutive threads take consecutive rows of A.
__global__ void __launch_bounds__(256) dense_sparse_kernel(int m, DView A, CscView B, DView C, int accumulate) {
    const int j = blockIdx.x;
    const int p0 = B.colptr[j], p1 = B.colptr[j + 1];
    const bool copy = p1 - p0 == 1 && B.vals[p0] == 1.0;
    for (long long r = (long long)blockIdx.y * blockDim.x + threadIdx.x; r < m; r += (long long)gridDim.y * blockDim.x) {
        const double* a = A.p + r * A.rs;
        double acc;
        if (copy) {
            acc = a[(long long)B.rowidx[p0] * A.cs];
        } else {
            acc = 0.0;
            for (int p = p0; p < p1; ++p) acc = __dadd_rn(acc, __dmul_rn(B.vals[p], a[(long long)B.rowidx[p] * A.cs]));
        }
        double* o = C.p + r * C.rs + (long long)j * C.cs;
        *o = put(o, acc, accumulate);
    }
}

// LibMatrixMult.multSparseDense (LibMatrixMult.scala:43-77) with the row offset of B read as `bk` (the reference reads `bi`
// at :60): C(r, i) = sum over k ascending of B(k, i) * A(r, k), the order of the corrected loop.  Row r of the CSR copy
// lists the k of row r ascending.  Consecutive threads take consecutive rows of C.
__global__ void __launch_bounds__(128) sparse_dense_kernel(CsrView A, int n, DView B, DView C, int accumulate) {
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= A.rows) return;
    const int q0 = A.rowptr[r], q1 = A.rowptr[r + 1];
    for (long long i = blockIdx.y; i < n; i += gridDim.y) {
        const double* b = B.p + i * B.cs;
        double acc = 0.0;
        for (int q = q0; q < q1; ++q) acc = __dadd_rn(acc, __dmul_rn(b[(long long)A.colidx[q] * B.rs], A.vals[q]));
        double* o = C.p + r * C.rs + i * C.cs;
        *o = put(o, acc, accumulate);
    }
}

// SparseMatrix.multiply (Matrices.scala:129-152): for each stored k of B(:, j) in order, C(:, j) += B(k, j) * A(:, k) over the
// stored rows of A(:, k).  One warp owns one column j and one chunk of SPG_CHUNK rows, accumulated in shared memory.  Within
// one k the rows are distinct (strictly increasing), so the lanes never meet; __syncwarp orders successive k.
constexpr int SPG_CHUNK = 1024;
constexpr int SPG_WARPS = 4;

__device__ __forceinline__ int lower_bound(const int* a, int lo, int hi, int key) {
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (a[mid] < key) lo = mid + 1; else hi = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(32 * SPG_WARPS) spgemm_kernel(CscView A, CscView B, DView C, int nchunks, long long ntasks,
                                                                int accumulate) {
    __shared__ double acc_s[SPG_WARPS][SPG_CHUNK];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long task = (long long)blockIdx.x * SPG_WARPS + warp;
    if (task >= ntasks) return;                      // warp-uniform
    const int j = (int)(task / nchunks), r0 = (int)(task % nchunks) * SPG_CHUNK;
    const int len = min(SPG_CHUNK, A.rows - r0);
    double* acc = acc_s[warp];
    for (int r = lane; r < len; r += 32) acc[r] = 0.0;
    __syncwarp();
    const int p1 = B.colptr[j + 1];
    for (int p = B.colptr[j]; p < p1; ++p) {
        const int k = B.rowidx[p];
        const double bv = B.vals[p];
        int lo = A.colptr[k], hi = A.colptr[k + 1];
        if (nchunks > 1) {
            lo = lower_bound(A.rowidx, lo, hi, r0);
            hi = lower_bound(A.rowidx, lo, hi, r0 + len);
        }
        for (int q = lo + lane; q < hi; q += 32) {
            const int r = A.rowidx[q] - r0;
            acc[r] = __dadd_rn(acc[r], __dmul_rn(bv, A.vals[q]));
        }
        __syncwarp();
    }
    for (int r = lane; r < len; r += 32) {
        double* o = C.p + (long long)(r0 + r) * C.rs + (long long)j * C.cs;
        *o = put(o, acc[r], accumulate);
    }
}

// ---- CSR copy: count per row, scan, scatter, then sort each row's short segment by column (the scatter's slot order
//      depends on atomic timing; after the sort the copy is a function of the CSC block alone) ----
__global__ void csr_count_kernel(const int* rowidx, long long nnz, int* counts) {
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < nnz; p += (long long)gridDim.x * blockDim.x)
        atomicAdd(&counts[rowidx[p]], 1);
}

// In-place inclusive prefix sum of a[0, len) by one CTA (integer: exact in any order).
__global__ void __launch_bounds__(1024) scan_inplace_kernel(int* a, long long len) {
    __shared__ long long part[1024];
    const long long per = (len + 1023) / 1024;
    const long long b = threadIdx.x * per, e = min(len, b + per);
    long long s = 0;
    for (long long i = b; i < e; ++i) s += a[i];
    part[threadIdx.x] = s;
    __syncthreads();
    for (int off = 1; off < 1024; off <<= 1) {
        const long long v = threadIdx.x >= off ? part[threadIdx.x - off] : 0;
        __syncthreads();
        part[threadIdx.x] += v;
        __syncthreads();
    }
    long long run = threadIdx.x ? part[threadIdx.x - 1] : 0;
    for (long long i = b; i < e; ++i) {
        run += a[i];
        a[i] = (int)run;
    }
}

__global__ void csr_scatter_kernel(CscView S, long long nnz, int* cursor, int* colidx, double* vals) {
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < nnz; p += (long long)gridDim.x * blockDim.x) {
        // column of entry p: the last k with colptr[k] <= p
        int lo = 0, hi = S.cols;
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if (S.colptr[mid] <= p) lo = mid; else hi = mid;
        }
        const int pos = atomicAdd(&cursor[S.rowidx[p]], 1);
        colidx[pos] = lo;
        vals[pos] = S.vals[p];
    }
}

__global__ void csr_sort_kernel(int rows, const int* rowptr, int* colidx, double* vals) {
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    const int q0 = rowptr[r], q1 = rowptr[r + 1];
    for (int q = q0 + 1; q < q1; ++q) {
        const int c = colidx[q];
        const double v = vals[q];
        int t = q - 1;
        while (t >= q0 && colidx[t] > c) {
            colidx[t + 1] = colidx[t];
            vals[t + 1] = vals[t];
            --t;
        }
        colidx[t + 1] = c;
        vals[t + 1] = v;
    }
}

// ---- sparse generator: rows of each column by selection sampling (Knuth, Algorithm S) ----
__device__ __forceinline__ unsigned long long xs_step(unsigned long long s) {
    s ^= s << 21;
    s ^= s >> 35;
    s ^= s << 4;
    return s;
}

// Column j jumps straight to stream position first + j*rows (two XORShift steps per position) and takes row t when
// x * (rows - t) < q * 2^53, x the 53-bit integer behind that position's nextDouble and q the rows still needed: select with
// probability q / (rows - t), in exact 128-bit integer arithmetic.  When q == rows - t the test always passes, so every
// column gets exactly s sorted rows.
__global__ void __launch_bounds__(128) sample_rows_kernel(int rows, int cols, int s, unsigned long long state0,
                                                          unsigned long long first, const unsigned long long* tab,
                                                          int* colptr, int* rowidx) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j > cols) return;
    colptr[j] = j * s;
    if (j == cols || s == 0) return;
    unsigned long long st = state0;
    unsigned long long steps = 2ull * (first + (unsigned long long)j * rows);
    for (int lv = 0; steps; ++lv, steps >>= 1) {
        if (steps & 1ull) {
            unsigned long long t = 0, x = st;
            while (x) {
                t ^= tab[lv * 64 + __ffsll((long long)x) - 1];
                x &= x - 1;
            }
            st = t;
        }
    }
    int* out = rowidx + (long long)j * s;
    int q = s;
    for (int t = 0; q > 0; ++t) {
        st = xs_step(st);
        const unsigned long long hi26 = st & ((1ull << 26) - 1);
        st = xs_step(st);
        const unsigned long long lo27 = st & ((1ull << 27) - 1);
        const unsigned long long x = (hi26 << 27) + lo27;
        const unsigned long long w = (unsigned long long)(rows - t);
        const unsigned long long plo = x * w, phi = __umul64hi(x, w);
        const unsigned long long qhi = (unsigned long long)q >> 11, qlo = (unsigned long long)q << 53;
        if (phi < qhi || (phi == qhi && plo < qlo)) {
            out[s - q] = t;
            --q;
        }
    }
}

}  // namespace

cudaError_t csc_to_dense(const CscView& S, DView out, cudaStream_t st) {
    if (S.rows <= 0 || S.cols <= 0) return cudaSuccess;
    csc_to_dense_kernel<<<S.cols, 256, 0, st>>>(S, out);
    return launched();
}

cudaError_t spmm_dense_sparse(int m, DView A, const CscView& B, DView C, bool accumulate, cudaStream_t st) {
    if (m <= 0 || B.cols <= 0) return cudaSuccess;
    const dim3 grid(B.cols, (unsigned)std::min<long long>((m + 255) / 256, 65535));
    dense_sparse_kernel<<<grid, 256, 0, st>>>(m, A, B, C, accumulate ? 1 : 0);
    return launched();
}

cudaError_t csc_to_csr(const CscView& S, long long nnz, int* rowptr, int* colidx, double* vals, cudaStream_t st) {
    cudaError_t e = cudaMemsetAsync(rowptr, 0, sizeof(int) * ((size_t)S.rows + 1), st);
    if (e != cudaSuccess || S.rows <= 0 || nnz <= 0) return e;
    const int g = (int)std::min<long long>((nnz + 255) / 256, 4096);
    csr_count_kernel<<<g, 256, 0, st>>>(S.rowidx, nnz, rowptr + 1);
    if ((e = launched()) != cudaSuccess) return e;
    scan_inplace_kernel<<<1, 1024, 0, st>>>(rowptr + 1, S.rows);
    if ((e = launched()) != cudaSuccess) return e;
    StreamBuffer cursor;
    if ((e = cursor.alloc(sizeof(int) * (size_t)S.rows, st)) != cudaSuccess) return e;
    e = cudaMemcpyAsync(cursor.as<int>(), rowptr, sizeof(int) * (size_t)S.rows, cudaMemcpyDeviceToDevice, st);
    if (e != cudaSuccess) return e;
    csr_scatter_kernel<<<g, 256, 0, st>>>(S, nnz, cursor.as<int>(), colidx, vals);
    if ((e = launched()) != cudaSuccess) return e;
    csr_sort_kernel<<<(S.rows + 127) / 128, 128, 0, st>>>(S.rows, rowptr, colidx, vals);
    return launched();
}

cudaError_t spmm_sparse_dense(const CsrView& A, int n, DView B, DView C, bool accumulate, cudaStream_t st) {
    if (A.rows <= 0 || n <= 0) return cudaSuccess;
    const dim3 grid((unsigned)((A.rows + 127) / 128), (unsigned)std::min(n, 65535));
    sparse_dense_kernel<<<grid, 128, 0, st>>>(A, n, B, C, accumulate ? 1 : 0);
    return launched();
}

cudaError_t spgemm_dense_out(const CscView& A, const CscView& B, DView C, bool accumulate, cudaStream_t st) {
    if (A.rows <= 0 || B.cols <= 0) return cudaSuccess;
    const int nchunks = (A.rows + SPG_CHUNK - 1) / SPG_CHUNK;
    const long long ntasks = (long long)nchunks * B.cols;
    const long long blocks = (ntasks + SPG_WARPS - 1) / SPG_WARPS;
    if (blocks > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
    spgemm_kernel<<<(unsigned)blocks, 32 * SPG_WARPS, 0, st>>>(A, B, C, nchunks, ntasks, accumulate ? 1 : 0);
    return launched();
}

cudaError_t sparse_sample_rows(int rows, int cols, int s, unsigned long long state0, long long first, int* colptr,
                               int* rowidx, cudaStream_t st) {
    const unsigned long long* tab = nullptr;
    cudaError_t e = fill_jump_tables(&tab);
    if (e != cudaSuccess) return e;
    sample_rows_kernel<<<(cols + 1 + 127) / 128, 128, 0, st>>>(rows, cols, s, state0, (unsigned long long)first, tab,
                                                               colptr, rowidx);
    return launched();
}

}  // namespace mb

// SparseVecMatrix (matrix/SparseVecMatrix.scala): the sparse x sparse product of multiplySparse (:22-50) row by row
// (Gustavson), the dense-rows-to-CSR conversion of DenseVecMatrix.toSparseVecMatrix (DenseVecMatrix.scala:1333-1353) and
// the shared column set of randomSpaVecMatrix (rdd/RandomRDD.scala:136-159).
//
// Arithmetic of multiplySparse: a = (float)A(i,k), b = (float)B(k,j) (the JVM's d2f, __double2float_rn), p = a * b
// rounded to float (__fmul_rn); C(i,j) is the first product, then each later one added with __fadd_rn, in the stored
// order of A's row i (k ascending).  No fused multiply-add, no atomic ever combines values, no flush to zero.  Within one
// k step the group of threads takes B(k, :), whose columns are distinct, so each accumulator is touched by one thread per
// step; a barrier between steps keeps the k order.  Slots are claimed with atomicCAS on keys only.  Every row's result is
// therefore a function of the row alone, whichever bin or launch handles it.
//
// Rows are binned on their product count u_i = sum over k of nnz(B(k, :)):
//   u_i <= MB_SPVEC_WARP_BOUND  one warp, open-addressing hash of 2 * bound slots in shared memory;
//   u_i <= MB_SPVEC_CTA_BOUND   one CTA, hash of 2 * bound slots;
//   above                       one CTA walking MB_SPVEC_WINDOW-column windows of the row's column range with float
//                               accumulators and a presence bitmap (the window comes out in column order); each
//                               window starts at the lowest column the row reaches at or after the previous one.
// Hash rows are sorted by column (bitonic, the empty key sorts last) before they are written.
#include "spvec.h"
#include "../../include/marlin_b200.h"
#include "launch.h"

#include <algorithm>
#include <climits>

namespace mb {
namespace {

constexpr int WARP_BOUND = MB_SPVEC_WARP_BOUND;
constexpr int CTA_BOUND = MB_SPVEC_CTA_BOUND;
constexpr int WINDOW = MB_SPVEC_WINDOW;
constexpr int WARP_SLOTS = 2 * WARP_BOUND;
constexpr int CTA_SLOTS = 2 * CTA_BOUND;
constexpr int ROW_WARPS = 8;          // warps (rows) per CTA of the warp bin
constexpr int CTA_THREADS = 256;
constexpr int WORDS_PER_THREAD = WINDOW / 32 / CTA_THREADS;
constexpr int EMPTY = INT_MAX;        // column ids are below nCols <= 2^31 - 1
static_assert(WINDOW % (32 * CTA_THREADS) == 0, "a window is a whole number of bitmap words per thread");
static_assert((WARP_SLOTS & (WARP_SLOTS - 1)) == 0 && (CTA_SLOTS & (CTA_SLOTS - 1)) == 0, "hash tables are powers of two");

__device__ __forceinline__ int lower_col(const int* a, int lo, int hi, int key) {
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (a[mid] < key) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// Per row: the bin, the candidate column range.  One warp per row; rows with no product get a count of 0 and no bin.
__global__ void __launch_bounds__(256) spvec_bound_kernel(CsrView A, CsrView B, int* lists, int* bin_size,
                                                          int2* range) {
    const int lane = threadIdx.x & 31;
    const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (i >= A.rows) return;
    long long u = 0;
    int lo = INT_MAX, hi = -1;
    const int q1 = A.rowptr[i + 1];
    for (int q = A.rowptr[i] + lane; q < q1; q += 32) {
        const int k = A.colidx[q];
        const int b0 = B.rowptr[k], b1 = B.rowptr[k + 1];
        if (b1 > b0) {
            u += b1 - b0;
            lo = min(lo, B.colidx[b0]);
            hi = max(hi, B.colidx[b1 - 1]);
        }
    }
    for (int off = 16; off; off >>= 1) {
        u += __shfl_xor_sync(0xffffffffu, u, off);
        lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, off));
        hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, off));
    }
    if (lane) return;
    range[i] = make_int2(lo, hi);
    if (u == 0) return;
    const int bin = u <= WARP_BOUND ? 0 : (u <= CTA_BOUND ? 1 : 2);
    lists[bin * (long long)A.rows + atomicAdd(&bin_size[bin], 1)] = (int)i;
}

// Column c into the hash (mask + 1 slots); NUMERIC: its value starts from p or adds p.
template <bool NUMERIC>
__device__ __forceinline__ void hash_put(int* keys, float* vals, int mask, int c, float p) {
    // the high bits of the Fibonacci product: they depend on every bit of c, so strided column ids spread out
    unsigned h = ((unsigned)c * 2654435761u) >> (32 - __popc(mask));
    while (true) {
        int k = *reinterpret_cast<volatile int*>(&keys[h]);
        if (k == EMPTY) {
            k = atomicCAS(&keys[h], EMPTY, c);
            if (k == EMPTY) {
                if (NUMERIC) vals[h] = p;
                return;
            }
        }
        if (k == c) {
            if (NUMERIC) vals[h] = __fadd_rn(vals[h], p);
            return;
        }
        h = (h + 1) & (unsigned)mask;
    }
}

// Ascending bitonic sort of N (key, value) slots by the threads tid = 0 .. nthreads-1 of a group; sync() is the group's
// barrier.  Keys are distinct (EMPTY repeats, but its values are never read).
template <int N, bool NUMERIC, class Sync>
__device__ __forceinline__ void bitonic_sort(int* keys, float* vals, int tid, int nthreads, Sync sync) {
    for (int size = 2; size <= N; size <<= 1)
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int t = tid; t < N / 2; t += nthreads) {
                const int lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
                const bool up = (lo & size) == 0;
                const int ka = keys[lo], kb = keys[hi];
                if ((ka > kb) == up) {
                    keys[lo] = kb;
                    keys[hi] = ka;
                    if (NUMERIC) {
                        const float v = vals[lo];
                        vals[lo] = vals[hi];
                        vals[hi] = v;
                    }
                }
            }
            sync();
        }
}

// The products of row i into the hash of a group (tid / nthreads; sync() is its barrier), in k order.
template <bool NUMERIC, class Sync>
__device__ __forceinline__ void accumulate_row(const CsrView& A, const CsrView& B, int i, int* keys, float* vals, int mask,
                                               int tid, int nthreads, Sync sync) {
    const int q1 = A.rowptr[i + 1];
    for (int q = A.rowptr[i]; q < q1; ++q) {
        const int k = A.colidx[q];
        const float a = NUMERIC ? __double2float_rn(A.vals[q]) : 0.0f;
        const int b1 = B.rowptr[k + 1];
        for (int p = B.rowptr[k] + tid; p < b1; p += nthreads)
            hash_put<NUMERIC>(keys, vals, mask, B.colidx[p], NUMERIC ? __fmul_rn(a, __double2float_rn(B.vals[p])) : 0.0f);
        sync();
    }
}

// Warp bin: one warp per row.  Symbolic (NUMERIC = false): rowptr[i + 1] = the row's distinct columns.  Numeric: the
// sorted row at rowptr[i].
template <bool NUMERIC>
__global__ void __launch_bounds__(32 * ROW_WARPS) spvec_warp_kernel(CsrView A, CsrView B, const int* list, int nrows,
                                                                    int* rowptr, int* colidx, double* vals) {
    __shared__ int keys_s[ROW_WARPS][WARP_SLOTS];
    __shared__ float vals_s[NUMERIC ? ROW_WARPS : 1][NUMERIC ? WARP_SLOTS : 1];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const long long t = (long long)blockIdx.x * ROW_WARPS + w;
    if (t >= nrows) return;                          // warp-uniform
    const int i = list[t];
    int* keys = keys_s[w];
    float* acc = vals_s[NUMERIC ? w : 0];
    for (int s = lane; s < WARP_SLOTS; s += 32) keys[s] = EMPTY;
    __syncwarp();
    auto sync = [] { __syncwarp(); };
    accumulate_row<NUMERIC>(A, B, i, keys, acc, WARP_SLOTS - 1, lane, 32, sync);
    if (!NUMERIC) {
        int n = 0;
        for (int s = lane; s < WARP_SLOTS; s += 32) n += keys[s] != EMPTY;
        n = __reduce_add_sync(0xffffffffu, n);
        if (lane == 0) rowptr[i + 1] = n;
        return;
    }
    bitonic_sort<WARP_SLOTS, NUMERIC>(keys, acc, lane, 32, sync);
    const int o = rowptr[i], n = rowptr[i + 1] - o;
    for (int s = lane; s < n; s += 32) {
        colidx[o + s] = keys[s];
        vals[o + s] = (double)acc[s];
    }
}

// CTA bin: one CTA per row, CTA_SLOTS keys (+ values) in dynamic shared memory.
template <bool NUMERIC>
__global__ void __launch_bounds__(CTA_THREADS) spvec_cta_kernel(CsrView A, CsrView B, const int* list, int* rowptr,
                                                                int* colidx, double* vals) {
    extern __shared__ int smem_i[];
    __shared__ int count;
    int* keys = smem_i;
    float* acc = reinterpret_cast<float*>(smem_i + CTA_SLOTS);
    const int i = list[blockIdx.x];
    if (threadIdx.x == 0) count = 0;
    for (int s = threadIdx.x; s < CTA_SLOTS; s += CTA_THREADS) keys[s] = EMPTY;
    __syncthreads();
    auto sync = [] { __syncthreads(); };
    accumulate_row<NUMERIC>(A, B, i, keys, acc, CTA_SLOTS - 1, threadIdx.x, CTA_THREADS, sync);
    if (!NUMERIC) {
        int n = 0;
        for (int s = threadIdx.x; s < CTA_SLOTS; s += CTA_THREADS) n += keys[s] != EMPTY;
        n = __reduce_add_sync(0xffffffffu, n);
        if ((threadIdx.x & 31) == 0) atomicAdd(&count, n);      // integer: exact in any order
        __syncthreads();
        if (threadIdx.x == 0) rowptr[i + 1] = count;
        return;
    }
    bitonic_sort<CTA_SLOTS, NUMERIC>(keys, acc, threadIdx.x, CTA_THREADS, sync);
    const int o = rowptr[i], n = rowptr[i + 1] - o;
    for (int s = threadIdx.x; s < n; s += CTA_THREADS) {
        colidx[o + s] = keys[s];
        vals[o + s] = (double)acc[s];
    }
}

// Window bin: one CTA per row walks [range.x, range.y] in windows of WINDOW columns.  Per window and k step the threads
// take B(k, :)'s columns inside the window (binary search of the sorted row); atomicOr on the presence bitmap tells a
// thread whether its column already holds a value.  Each window is then emitted in column order from the bitmap.
template <bool NUMERIC>
__global__ void __launch_bounds__(CTA_THREADS) spvec_window_kernel(CsrView A, CsrView B, const int* list, const int2* range,
                                                                   int* rowptr, int* colidx, double* vals) {
    extern __shared__ unsigned smem_u[];
    unsigned* bits = smem_u;
    int* part = reinterpret_cast<int*>(bits + WINDOW / 32);
    float* acc = reinterpret_cast<float*>(part + CTA_THREADS);
    const int i = list[blockIdx.x];
    const int2 r = range[i];
    const int q0 = A.rowptr[i], q1 = A.rowptr[i + 1];
    int out = NUMERIC ? rowptr[i] : 0;
    for (long long w0 = r.x; w0 <= r.y;) {
        const int w1 = (int)min((long long)r.y + 1, w0 + WINDOW);
        long long next = LLONG_MAX;                  // the lowest column at or after w1: where the next window starts
        for (int x = threadIdx.x; x < WINDOW / 32; x += CTA_THREADS) bits[x] = 0u;
        __syncthreads();
        for (int q = q0; q < q1; ++q) {
            const int k = A.colidx[q];
            const int end = B.rowptr[k + 1];
            const int b0 = lower_col(B.colidx, B.rowptr[k], end, (int)w0);
            const int b1 = lower_col(B.colidx, b0, end, w1);
            if (b1 < end) next = min(next, (long long)B.colidx[b1]);
            if (b0 == b1) continue;                  // block-uniform
            const float a = NUMERIC ? __double2float_rn(A.vals[q]) : 0.0f;
            for (int p = b0 + threadIdx.x; p < b1; p += CTA_THREADS) {
                const int c = B.colidx[p] - (int)w0;
                const unsigned bit = 1u << (c & 31);
                const unsigned old = atomicOr(&bits[c >> 5], bit);
                if (NUMERIC) {
                    const float prod = __fmul_rn(a, __double2float_rn(B.vals[p]));
                    acc[c] = (old & bit) ? __fadd_rn(acc[c], prod) : prod;
                }
            }
            __syncthreads();
        }
        int cnt = 0;
        for (int x = 0; x < WORDS_PER_THREAD; ++x) cnt += __popc(bits[threadIdx.x * WORDS_PER_THREAD + x]);
        part[threadIdx.x] = cnt;
        __syncthreads();
        for (int off = 1; off < CTA_THREADS; off <<= 1) {
            const int v = threadIdx.x >= off ? part[threadIdx.x - off] : 0;
            __syncthreads();
            part[threadIdx.x] += v;
            __syncthreads();
        }
        if (NUMERIC) {
            int o = out + part[threadIdx.x] - cnt;
            for (int x = 0; x < WORDS_PER_THREAD; ++x) {
                const int word = threadIdx.x * WORDS_PER_THREAD + x;
                for (unsigned m = bits[word]; m; m &= m - 1) {
                    const int c = word * 32 + __ffs(m) - 1;
                    colidx[o] = (int)w0 + c;
                    vals[o] = (double)acc[c];
                    ++o;
                }
            }
        }
        out += part[CTA_THREADS - 1];
        __syncthreads();                             // the next window clears bits and part
        w0 = next;                                   // windows holding no column are skipped
    }
    if (!NUMERIC && threadIdx.x == 0) rowptr[i + 1] = out;
}

// In-place inclusive prefix sum of a[0, len) by one CTA, as scan_inplace_kernel, plus the int64 total.
__global__ void __launch_bounds__(1024) spvec_scan_kernel(int* a, long long len, long long* total) {
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
    if (threadIdx.x == 1023) *total = part[1023];
}

// toSparseVecMatrix: one warp per row, entries != 0.0 (NaN kept, +-0.0 dropped) in column order.  COMPACT = false counts
// into rowptr[i + 1].
template <bool COMPACT>
__global__ void __launch_bounds__(256) dense_rows_kernel(DView D, int rows, int cols, int* rowptr, int* colidx,
                                                         double* vals) {
    const int lane = threadIdx.x & 31;
    const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (i >= rows) return;
    const double* row = D.p + i * D.rs;
    int o = COMPACT ? rowptr[i] : 0;
    for (int c0 = 0; c0 < cols; c0 += 32) {
        const int c = c0 + lane;
        const double v = c < cols ? row[(long long)c * D.cs] : 0.0;
        const bool keep = v != 0.0;
        const unsigned m = __ballot_sync(0xffffffffu, keep);
        if (COMPACT && keep) {
            const int pos = o + __popc(m & ((1u << lane) - 1u));
            colidx[pos] = c;
            vals[pos] = v;
        }
        o += __popc(m);
    }
    if (!COMPACT && lane == 0) rowptr[i + 1] = o;
}

__global__ void spvec_replicate_kernel(int rows, int s, int* rowptr, int* colidx) {
    const long long n = (long long)rows * s;
    for (long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x; x < n || x <= rows;
         x += (long long)gridDim.x * blockDim.x) {
        if (x <= rows) rowptr[x] = (int)(x * s);
        if (x >= s && x < n) colidx[x] = colidx[x % s];
    }
}

cudaError_t scan(int* rowptr, int rows, long long* total_d, long long* total, cudaStream_t st) {
    spvec_scan_kernel<<<1, 1024, 0, st>>>(rowptr + 1, rows, total_d);
    cudaError_t e = launched();
    if (e == cudaSuccess) e = cudaMemcpyAsync(total, total_d, sizeof(long long), cudaMemcpyDeviceToHost, st);
    return e == cudaSuccess ? cudaStreamSynchronize(st) : e;
}

unsigned warps_grid(long long rows) { return (unsigned)((rows * 32 + 255) / 256); }

}  // namespace

cudaError_t spvec_count(const CsrView& A, const CsrView& B, int* rowptr, long long* total, SpvecWork* w, cudaStream_t st) {
    *total = 0;
    cudaError_t e = cudaMemsetAsync(rowptr, 0, sizeof(int) * ((size_t)A.rows + 1), st);
    if (e != cudaSuccess || A.rows == 0) return e;
    if ((e = w->lists.alloc(sizeof(int) * 3 * (size_t)A.rows, st)) != cudaSuccess) return e;
    if ((e = w->range.alloc(sizeof(int2) * (size_t)A.rows, st)) != cudaSuccess) return e;
    if ((e = w->bin_size.alloc(32, st)) != cudaSuccess) return e;
    int *lists = w->lists.as<int>(), *bin_size = w->bin_size.as<int>();
    if ((e = cudaMemsetAsync(bin_size, 0, 32, st)) != cudaSuccess) return e;
    spvec_bound_kernel<<<warps_grid(A.rows), 256, 0, st>>>(A, B, lists, bin_size, w->range.as<int2>());
    if ((e = launched()) != cudaSuccess) return e;
    if ((e = cudaMemcpyAsync(w->bins, bin_size, sizeof(w->bins), cudaMemcpyDeviceToHost, st)) != cudaSuccess) return e;
    if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return e;
    const long long n = A.rows;
    if (w->bins[0]) {
        spvec_warp_kernel<false><<<(w->bins[0] + ROW_WARPS - 1) / ROW_WARPS, 32 * ROW_WARPS, 0, st>>>(A, B, lists, w->bins[0],
                                                                                                      rowptr, nullptr, nullptr);
        if ((e = launched()) != cudaSuccess) return e;
    }
    if (w->bins[1]) {
        spvec_cta_kernel<false><<<w->bins[1], CTA_THREADS, sizeof(int) * CTA_SLOTS, st>>>(A, B, lists + n, rowptr, nullptr,
                                                                                          nullptr);
        if ((e = launched()) != cudaSuccess) return e;
    }
    if (w->bins[2]) {
        const size_t smem = sizeof(unsigned) * (WINDOW / 32) + sizeof(int) * CTA_THREADS;
        spvec_window_kernel<false><<<w->bins[2], CTA_THREADS, smem, st>>>(A, B, lists + 2 * n, w->range.as<int2>(), rowptr, nullptr,
                                                                          nullptr);
        if ((e = launched()) != cudaSuccess) return e;
    }
    return scan(rowptr, A.rows, reinterpret_cast<long long*>(bin_size + 4), total, st);
}

cudaError_t spvec_fill(const CsrView& A, const CsrView& B, const SpvecWork& w, const int* rowptr, int* colidx, double* vals,
                       cudaStream_t st) {
    const long long n = A.rows;
    int* rp = const_cast<int*>(rowptr);
    const int* lists = w.lists.as<int>();
    cudaError_t e;
    if (w.bins[0]) {
        spvec_warp_kernel<true><<<(w.bins[0] + ROW_WARPS - 1) / ROW_WARPS, 32 * ROW_WARPS, 0, st>>>(A, B, lists, w.bins[0], rp,
                                                                                                    colidx, vals);
        if ((e = launched()) != cudaSuccess) return e;
    }
    if (w.bins[1]) {
        const size_t smem = (sizeof(int) + sizeof(float)) * CTA_SLOTS;
        if ((e = cudaFuncSetAttribute(spvec_cta_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess)
            return e;
        spvec_cta_kernel<true><<<w.bins[1], CTA_THREADS, smem, st>>>(A, B, lists + n, rp, colidx, vals);
        if ((e = launched()) != cudaSuccess) return e;
    }
    if (w.bins[2]) {
        const size_t smem = sizeof(unsigned) * (WINDOW / 32) + sizeof(int) * CTA_THREADS + sizeof(float) * WINDOW;
        if ((e = cudaFuncSetAttribute(spvec_window_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess)
            return e;
        spvec_window_kernel<true><<<w.bins[2], CTA_THREADS, smem, st>>>(A, B, lists + 2 * n, w.range.as<int2>(), rp, colidx, vals);
        return launched();
    }
    return cudaSuccess;
}

cudaError_t dense_rows_count(DView D, int rows, int cols, int* rowptr, long long* total, cudaStream_t st) {
    *total = 0;
    cudaError_t e = cudaMemsetAsync(rowptr, 0, sizeof(int) * ((size_t)rows + 1), st);
    if (e != cudaSuccess || rows == 0) return e;
    StreamBuffer total_d;
    if ((e = total_d.alloc(sizeof(long long), st)) != cudaSuccess) return e;
    dense_rows_kernel<false><<<warps_grid(rows), 256, 0, st>>>(D, rows, cols, rowptr, nullptr, nullptr);
    e = launched();
    return e == cudaSuccess ? scan(rowptr, rows, total_d.as<long long>(), total, st) : e;
}

cudaError_t dense_rows_compact(DView D, int rows, int cols, const int* rowptr, int* colidx, double* vals, cudaStream_t st) {
    if (rows == 0) return cudaSuccess;
    dense_rows_kernel<true><<<warps_grid(rows), 256, 0, st>>>(D, rows, cols, const_cast<int*>(rowptr), colidx, vals);
    return launched();
}

cudaError_t spvec_replicate_columns(int rows, int s, int* rowptr, int* colidx, cudaStream_t st) {
    const long long n = std::max<long long>((long long)rows * s, (long long)rows + 1);
    spvec_replicate_kernel<<<(unsigned)std::min<long long>((n + 255) / 256, 4096), 256, 0, st>>>(rows, s, rowptr, colidx);
    return launched();
}

}  // namespace mb

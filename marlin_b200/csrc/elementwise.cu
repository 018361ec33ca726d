// HBM-bound block kernels: add / subtract / scalar ops / Hadamard / transpose / copy / sum and the
// on-device XORShift input generator.  All of these stream each element once, so the design is
// 128-bit vectorised global accesses, enough bytes in flight per SM, no shared memory except for
// the transpose (which needs it to make both the load and the store side coalesced).
//
// Reference semantics: matrix/SubMatrix.scala:41-85,123-131 (Breeze + - / * on BDM),
// matrix/BlockMatrix.scala:414-452 (subtractBy/divideBy), :467-472 (sum), :494-500 (dotProduct =
// Hadamard), :514-523 (transpose = denseBlock.t.copy), utils/RandomDataGenerator.scala:53-65,113-131.
#include "elementwise.h"
#include "launch.h"
#include "ptx.cuh"
#include <cuda_bf16.h>
#include <atomic>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <vector>

namespace mb {

namespace {

constexpr int EW_THREADS = 256;

__device__ __forceinline__ double apply_bin(int op, double a, double b) {
    switch (op) {
        case EW_ADD: return __dadd_rn(a, b);
        case EW_SUB: return __dsub_rn(a, b);
        default: return __dmul_rn(a, b);
    }
}
// alpha*a + beta with two roundings (the JVM never fuses); EW_DIV: a / s ; EW_RDIV: s / a
__device__ __forceinline__ double apply_un(int op, double a, double alpha, double beta) {
    switch (op) {
        case EW_AXPB: return __dadd_rn(__dmul_rn(alpha, a), beta);
        case EW_DIV: return __ddiv_rn(a, alpha);
        case EW_RDIV: return __ddiv_rn(alpha, a);
        case EW_FILL: return beta;
        default: return a;
    }
}

// ---- flat (packed, same orientation) fast paths: 128-bit accesses, 4 independent loads in flight ----
// Flat (packed, same orientation) fast paths.  One CTA per contiguous 16 KiB tile (256 threads x 4 vectors of 16 B, all
// four loads issued before the first store), plain ld/st.global, non-persistent: the block scheduler walks the array in
// address order.  An earlier persistent grid-stride + ld.nc/st.cs variant was slower and was dropped.
template <int OP>
__global__ void __launch_bounds__(EW_THREADS) binary_flat_kernel(const double2* a, const double2* b, double2* o,
                                                                long long n2) {      // o may alias a or b exactly (in-place)
    constexpr int TILE = EW_THREADS * 4;
    const long long base = (long long)blockIdx.x * TILE + threadIdx.x;
    if (base + 3 * EW_THREADS < n2) {
        double2 x[4], y[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) { x[u] = a[base + u * EW_THREADS]; y[u] = b[base + u * EW_THREADS]; }
#pragma unroll
        for (int u = 0; u < 4; ++u)
            o[base + u * EW_THREADS] = make_double2(apply_bin(OP, x[u].x, y[u].x), apply_bin(OP, x[u].y, y[u].y));
    } else {
        for (int u = 0; u < 4; ++u) {
            const long long i = base + u * EW_THREADS;
            if (i < n2) {
                const double2 x = a[i], y = b[i];
                o[i] = make_double2(apply_bin(OP, x.x, y.x), apply_bin(OP, x.y, y.y));
            }
        }
    }
}

template <int OP>
__global__ void __launch_bounds__(EW_THREADS) unary_flat_kernel(const double2* a, double2* o, long long n2, double alpha,
                                                               double beta) {          // o may alias a exactly (in-place)
    constexpr int TILE = EW_THREADS * 4;
    const long long base = (long long)blockIdx.x * TILE + threadIdx.x;
    if (base + 3 * EW_THREADS < n2) {
        double2 x[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) x[u] = a[base + u * EW_THREADS];
#pragma unroll
        for (int u = 0; u < 4; ++u)
            o[base + u * EW_THREADS] = make_double2(apply_un(OP, x[u].x, alpha, beta), apply_un(OP, x[u].y, alpha, beta));
    } else {
        for (int u = 0; u < 4; ++u) {
            const long long i = base + u * EW_THREADS;
            if (i < n2) {
                const double2 x = a[i];
                o[i] = make_double2(apply_un(OP, x.x, alpha, beta), apply_un(OP, x.y, alpha, beta));
            }
        }
    }
}

// ---- general strided path (views with ld != rows, odd sizes, mixed orientation) ----
// element (r,c) of a view: base[r*rs + c*cs]
__global__ void binary_strided_kernel(int op, int rows, int cols, const double* a, long long ars, long long acs,
                                      const double* b, long long brs, long long bcs, double* o, long long ors,
                                      long long ocs) {
    const long long total = (long long)rows * cols;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total;
         e += (long long)gridDim.x * blockDim.x) {
        const long long r = e % rows, c = e / rows;
        const double x = a[r * ars + c * acs], y = b[r * brs + c * bcs];
        o[r * ors + c * ocs] = (op == EW_ADD) ? __dadd_rn(x, y) : (op == EW_SUB) ? __dsub_rn(x, y) : __dmul_rn(x, y);
    }
}
__global__ void unary_strided_kernel(int op, int rows, int cols, const double* a, long long ars, long long acs,
                                     double* o, long long ors, long long ocs, double alpha, double beta) {
    const long long total = (long long)rows * cols;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total;
         e += (long long)gridDim.x * blockDim.x) {
        const long long r = e % rows, c = e / rows;
        const double x = a[r * ars + c * acs];
        double v;
        if (op == EW_AXPB) v = __dadd_rn(__dmul_rn(alpha, x), beta);
        else if (op == EW_DIV) v = __ddiv_rn(x, alpha);
        else if (op == EW_RDIV) v = __ddiv_rn(alpha, x);
        else if (op == EW_FILL) v = beta;
        else v = x;
        o[r * ors + c * ocs] = v;
    }
}

// fp32 blocks (the C tiles of the bf16 path): same operators, strided form only
__global__ void binary_strided_f32_kernel(int op, int rows, int cols, const float* a, long long ars, long long acs,
                                          const float* b, long long brs, long long bcs, float* o, long long ors,
                                          long long ocs) {
    const long long total = (long long)rows * cols;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total;
         e += (long long)gridDim.x * blockDim.x) {
        const long long r = e % rows, c = e / rows;
        const float x = a[r * ars + c * acs], y = b[r * brs + c * bcs];
        o[r * ors + c * ocs] = (op == EW_ADD) ? __fadd_rn(x, y) : (op == EW_SUB) ? __fsub_rn(x, y) : __fmul_rn(x, y);
    }
}

// ---- transpose: out (cols x rows, ldo) = in (rows x cols, ldi)^T, both column-major ----
// 64x64 tile = 32x32 micro-blocks of 2x2 doubles.  Each thread loads a 2x2 micro-block with two
// 128-bit loads (two adjacent columns), transposes it in registers, parks it in shared memory and a
// different thread writes it with two 128-bit stores, so both HBM directions are fully coalesced.
// Shared-memory slot of 16B unit (rb, cb, half):  rb*64 + 16*(cb>>3) + 8*half + ((cb&7) ^ (rb&7))
// which is conflict-free for the column-wise writes and the row-wise reads.
constexpr int TT = 64;
// A CTA owns TT_SUB vertically adjacent 64x64 sub-tiles, so it reads 1 KiB runs per input column (all its loads are
// issued before its single barrier).  CTAs walk bands of TT_BAND tile columns, column-tile fastest inside a band, so
// the CTAs in flight write TT_BAND * 512 B runs per output column and read long runs per input column.
constexpr int TT_SUB = 2, TT_BAND = 8;
constexpr int TT_SMEM = TT_SUB * 32 * 64 * (int)sizeof(double2);
__global__ void __launch_bounds__(256) transpose_f64_tile_kernel(const double* __restrict__ in, long long ldi,
                                                                double* __restrict__ out, long long ldo, int rows,
                                                                int cols, int tiles_r, int tiles_c) {
    extern __shared__ double2 tile_all[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int band = blockIdx.x / (TT_BAND * tiles_r);
    const int rem = blockIdx.x - band * (TT_BAND * tiles_r);
    const int gw = min(TT_BAND, tiles_c - band * TT_BAND);       // last band may be narrower
    const int tc = band * TT_BAND + rem % gw;
    const int tr = rem / gw;
    const int c0 = tc * TT;
    // load phase: lane -> micro-row rb, warp -> micro-cols cb = warp + 8*i
#pragma unroll
    for (int sr = 0; sr < TT_SUB; ++sr) {
        double2* tile = tile_all + sr * (32 * 64);
        const int rb = lane;
        const int r = (tr * TT_SUB + sr) * TT + 2 * rb;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int cb = warp + 8 * i;
            const int c = c0 + 2 * cb;
            double2 v0 = make_double2(0.0, 0.0), v1 = v0;
            if (r < rows && c < cols) {   // rows, cols even -> whole micro-block in range
                v0 = *reinterpret_cast<const double2*>(in + r + (long long)c * ldi);
                v1 = *reinterpret_cast<const double2*>(in + r + (long long)(c + 1) * ldi);
            }
            const int base = rb * 64 + 16 * (cb >> 3) + ((cb & 7) ^ (rb & 7));
            tile[base] = make_double2(v0.x, v1.x);       // out column r   : in(r, c), in(r, c+1)
            tile[base + 8] = make_double2(v0.y, v1.y);   // out column r+1 : in(r+1, c), in(r+1, c+1)
        }
    }
    __syncthreads();
    // store phase
#pragma unroll
    for (int sr = 0; sr < TT_SUB; ++sr) {
        const double2* tile = tile_all + sr * (32 * 64);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int rb = warp + 8 * i;
            const int r = (tr * TT_SUB + sr) * TT + 2 * rb;
            const int cb = lane;
            const int c = c0 + 2 * cb;
#pragma unroll
            for (int half = 0; half < 2; ++half)
                if (r < rows && c < cols) {
                    const int base = rb * 64 + 16 * (cb >> 3) + ((cb & 7) ^ (rb & 7));
                    *reinterpret_cast<double2*>(out + c + (long long)(r + half) * ldo) = tile[base + 8 * half];
                }
        }
    }
}

// generic transpose (any alignment / odd sizes / any element type): 32x32 tile, scalar accesses
template <typename T>
__global__ void __launch_bounds__(256) transpose_generic_kernel(const T* __restrict__ in, long long ldi,
                                                               T* __restrict__ out, long long ldo, int rows, int cols) {
    __shared__ T tile[32][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int r0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int r = r0 + tx, c = c0 + ty + 8 * i;
        if (r < rows && c < cols) tile[ty + 8 * i][tx] = in[r + (long long)c * ldi];
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int c = c0 + tx, r = r0 + ty + 8 * i;
        if (r < rows && c < cols) out[c + (long long)r * ldo] = tile[tx][ty + 8 * i];
    }
}

// ---- sum: two-stage deterministic tree (fixed grid => run-to-run reproducible) ----
constexpr int SUM_BLOCKS = 16384;      // upper bound on stage-1 CTAs (one 16 KiB tile per CTA-iteration)
__device__ __forceinline__ double block_reduce_sum(double v) {
    __shared__ double warp_part[8];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) warp_part[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x < 8) t = warp_part[threadIdx.x];
    if (threadIdx.x < 32) {
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    }
    return t;
}
__global__ void __launch_bounds__(256) sum_strided_kernel(const double* __restrict__ a, int rows, int cols,
                                                         long long ld, double* __restrict__ partial) {
    const long long total = (long long)rows * cols;
    double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
    const bool packed_vec = (ld == rows) && ((reinterpret_cast<uintptr_t>(a) & 15) == 0);
    if (packed_vec) {
        // contiguous 16 KiB tiles, four independent 128-bit loads per thread and iteration (same shape as the flat
        // element-wise kernels); the tile -> CTA map and the in-thread order are fixed, so the sum is reproducible
        const long long n2 = total >> 1;
        const double2* a2 = reinterpret_cast<const double2*>(a);
        constexpr int TILE = 256 * 4;
        const long long num_tiles = (n2 + TILE - 1) / TILE;
        for (long long t = blockIdx.x; t < num_tiles; t += gridDim.x) {
            const long long base = t * TILE + threadIdx.x;
            if (base + 3 * 256 < n2) {
                const double2 v0 = a2[base], v1 = a2[base + 256], v2 = a2[base + 512], v3 = a2[base + 768];
                s0 += v0.x + v0.y; s1 += v1.x + v1.y; s2 += v2.x + v2.y; s3 += v3.x + v3.y;
            } else {
                for (int u = 0; u < 4; ++u) {
                    const long long i = base + u * 256;
                    if (i < n2) { const double2 v = a2[i]; s0 += v.x + v.y; }
                }
            }
        }
        if ((total & 1) && blockIdx.x == 0 && threadIdx.x == 0) s0 += a[total - 1];
    } else {
        for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total;
             e += (long long)gridDim.x * blockDim.x)
            s0 += a[(e % rows) + (e / rows) * ld];
    }
    const double t = block_reduce_sum((s0 + s1) + (s2 + s3));
    if (threadIdx.x == 0) partial[blockIdx.x] = t;
}
__global__ void __launch_bounds__(256) sum_final_kernel(const double* __restrict__ partial, int n, double* out) {
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) s += partial[i];
    const double t = block_reduce_sum(s);
    if (threadIdx.x == 0) *out = t;
}

// ---- dtype conversion (fp64 <-> bf16 / fp32), strided views ----
template <typename TI, typename TO>
__device__ __forceinline__ TO cvt(TI v);
template <> __device__ __forceinline__ double cvt<double, double>(double v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 cvt<double, __nv_bfloat16>(double v) { return __double2bfloat16(v); }
template <> __device__ __forceinline__ float cvt<double, float>(double v) { return __double2float_rn(v); }
template <> __device__ __forceinline__ double cvt<__nv_bfloat16, double>(__nv_bfloat16 v) { return (double)__bfloat162float(v); }
template <> __device__ __forceinline__ double cvt<float, double>(float v) { return (double)v; }
template <> __device__ __forceinline__ __nv_bfloat16 cvt<__nv_bfloat16, __nv_bfloat16>(__nv_bfloat16 v) { return v; }
template <> __device__ __forceinline__ float cvt<float, float>(float v) { return v; }
template <> __device__ __forceinline__ float cvt<__nv_bfloat16, float>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <> __device__ __forceinline__ __nv_bfloat16 cvt<float, __nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

template <typename TI, typename TO>
__global__ void convert_strided_kernel(int rows, int cols, const TI* a, long long ars, long long acs, TO* o,
                                       long long ors, long long ocs) {
    const long long total = (long long)rows * cols;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total;
         e += (long long)gridDim.x * blockDim.x) {
        const long long r = e % rows, c = e / rows;
        o[r * ors + c * ocs] = cvt<TI, TO>(a[r * ars + c * acs]);
    }
}

// ---- XORShift uniform generator (utils/RandomDataGenerator.scala:113-131) ----
// state' = s ^ (s<<21); ^= (>>>35); ^= (<<4).  The map is GF(2)-linear, so value i of a partition
// stream is reachable by a jump: state_i = T^(2i) * state_0 (nextDouble consumes two steps).
// g_jump[j] holds the 64 columns of T^(2^j); a chunk start is the product of the set bits of 2*first.

__device__ __forceinline__ unsigned long long xs_step(unsigned long long s) {
    s ^= s << 21;
    s ^= s >> 35;
    s ^= s << 4;
    return s;
}
__device__ unsigned long long g_jump[40][64];      // columns of T^(2^j), j = 0..39 (global memory: lane-parallel access)

// T^steps * s computed by a whole warp: lane l owns columns l and l+32 of each power-of-two matrix, the partial XORs
// are combined with shuffles.  ~25 instructions per set bit of `steps` instead of a 64-iteration serial loop.
__device__ __forceinline__ unsigned long long xs_jump_warp(unsigned long long s, unsigned long long steps, int lane) {
    for (int j = 0; j < 40 && steps; ++j, steps >>= 1) {
        if (steps & 1ull) {
            unsigned long long v = ((s >> lane) & 1ull) ? g_jump[j][lane] : 0ull;
            v ^= ((s >> (lane + 32)) & 1ull) ? g_jump[j][lane + 32] : 0ull;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v ^= __shfl_xor_sync(0xffffffffu, v, o);
            s = v;
        }
    }
    return s;
}

// One CTA = 256 threads x FILL_PER_THREAD consecutive values (512 KiB of output).  Thread t owns values
// [block_first + t*FILL_PER_THREAD, +FILL_PER_THREAD): long per-thread runs amortise the jump-ahead (one CTA-base jump by
// warp 0, a 3-level warp part done cooperatively, a <= 5-level lane part done serially, all from shared-memory tables),
// and the values go out in rounds of FILL_ROUND per thread through a padded shared-memory stage so that every store
// instruction writes whole 128-byte lines.
constexpr int FILL_PER_THREAD = 256;
constexpr int FILL_ROUND = 16;
constexpr int FILL_LVL0 = 9;        // thread offset = t * 2 * FILL_PER_THREAD steps = t << 9: table levels 9..16
__global__ void __launch_bounds__(256) fill_uniform_kernel(double* out, long long rs, long long cs, int rows, int cols,
                                                          int row_major, unsigned long long state0, long long first,
                                                          double lo, double hi, int block_offset) {
    __shared__ __align__(16) double stage[256][FILL_ROUND + 2];      // row stride 18 doubles: 16-byte aligned rows,
                                                                     // conflict-free 128-bit accesses per quarter warp
    __shared__ unsigned long long jump_s[8][64];
    __shared__ unsigned long long base_s;
    const long long total = (long long)rows * cols;
    const long long block_first = (long long)(blockIdx.x + block_offset) * 256 * FILL_PER_THREAD;
    if (block_first >= total) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int e = threadIdx.x; e < 8 * 64; e += 256) jump_s[e >> 6][e & 63] = g_jump[FILL_LVL0 + (e >> 6)][e & 63];
    if (warp == 0) {
        const unsigned long long b = xs_jump_warp(state0, 2ull * (unsigned long long)(first + block_first), lane);
        if (lane == 0) base_s = b;
    }
    __syncthreads();
    unsigned long long s = base_s;
    // warp part: bits 5..7 of the thread index -> levels FILL_LVL0+5 .. +7, one matrix-vector product per set bit by the
    // whole warp (lane l owns columns l and l+32)
#pragma unroll
    for (int j = 5; j < 8; ++j) {
        if ((warp >> (j - 5)) & 1) {
            unsigned long long v = ((s >> lane) & 1ull) ? jump_s[j][lane] : 0ull;
            v ^= ((s >> (lane + 32)) & 1ull) ? jump_s[j][lane + 32] : 0ull;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v ^= __shfl_xor_sync(0xffffffffu, v, o);
            s = v;
        }
    }
    // lane part: bits 0..4 -> levels FILL_LVL0 .. +4, serial (every lane has its own vector by now)
#pragma unroll 1
    for (int j = 0; j < 5; ++j) {
        if ((lane >> j) & 1) {
            unsigned long long t = 0, x = s;
            while (x) {
                t ^= jump_s[j][__ffsll((long long)x) - 1];
                x &= x - 1;
            }
            s = t;
        }
    }
    const double span = __dsub_rn(hi, lo);
    // storage contiguous in fill order (a row-major shard filled row-major, or a packed column-major block filled
    // column-major): linear index == storage index, no 64-bit divisions on the store path
    const bool linear = row_major ? (cs == 1 && rs == cols) : (rs == 1 && cs == rows);
    const int block_cnt = (int)min((long long)256 * FILL_PER_THREAD, total - block_first);     // values this CTA owns
    const int my_first = threadIdx.x * FILL_PER_THREAD;                                         // relative to block_first
    double* dst = out + block_first;
    const bool vec = linear && ((reinterpret_cast<uintptr_t>(dst) & 15) == 0);
#pragma unroll 1
    for (int round = 0; round < FILL_PER_THREAD / FILL_ROUND; ++round) {
        if (round * FILL_ROUND >= block_cnt) break;       // uniform: thread 0's run is the earliest, nothing left for anyone
        if (my_first + round * FILL_ROUND < block_cnt) {
#pragma unroll
            for (int v = 0; v < FILL_ROUND; v += 2) {
                double2 pr;
                {
                    s = xs_step(s);
                    const unsigned long long hi26 = s & ((1ull << 26) - 1);
                    s = xs_step(s);
                    const unsigned long long lo27 = s & ((1ull << 27) - 1);
                    pr.x = __dadd_rn(__dmul_rn(span, (double)((hi26 << 27) + lo27) * 0x1.0p-53), lo);
                }
                {
                    s = xs_step(s);
                    const unsigned long long hi26 = s & ((1ull << 26) - 1);
                    s = xs_step(s);
                    const unsigned long long lo27 = s & ((1ull << 27) - 1);
                    pr.y = __dadd_rn(__dmul_rn(span, (double)((hi26 << 27) + lo27) * 0x1.0p-53), lo);
                }
                *reinterpret_cast<double2*>(&stage[threadIdx.x][v]) = pr;
            }
        }
        __syncthreads();
        // pair p of the round: owner thread p / 8, its values 2*(p % 8), +1 -> 8 consecutive lanes write one 128-byte line
        if (vec) {
#pragma unroll
            for (int p = threadIdx.x; p < 256 * (FILL_ROUND / 2); p += 256) {
                const int owner = p >> 3, j = (p & 7) * 2;
                const int idx = owner * FILL_PER_THREAD + round * FILL_ROUND + j;
                if (idx + 1 < block_cnt) {
                    *reinterpret_cast<double2*>(dst + idx) = *reinterpret_cast<const double2*>(&stage[owner][j]);
                } else if (idx < block_cnt) {
                    dst[idx] = stage[owner][j];
                }
            }
        } else {
#pragma unroll 4
            for (int e = threadIdx.x; e < 256 * FILL_ROUND; e += 256) {
                const int owner = e / FILL_ROUND, j = e % FILL_ROUND;
                const int idx = owner * FILL_PER_THREAD + round * FILL_ROUND + j;
                if (idx < block_cnt) {
                    if (linear) {
                        dst[idx] = stage[owner][j];
                    } else {
                        const long long i = block_first + idx;
                        long long r, c;
                        if (row_major) { r = i / cols; c = i - r * cols; } else { c = i / rows; r = i - c * rows; }
                        out[r * rs + c * cs] = stage[owner][j];
                    }
                }
            }
        }
        __syncthreads();
    }
}

// ---- the fast path: a FULL CTA (65,536 values) of a linear, 16-byte aligned destination --------------------------
// Same stream positions, same values, fewer issue slots per value (the first version spent 57.7 thread instructions per
// value and was issue-bound):
//   * the XORShift step works on the two 32-bit halves and takes its left shifts from the multiplier — one IMAD.WIDE
//     yields (lo << k, lo >> (32-k)) and one IMAD folds in hi << k — so the fma pipe carries the shifts and the alu pipe
//     only the XORs (the shift counts arrive as kernel arguments, or the compiler turns them back into SHF);
//   * nextDouble = a * 2^-26 + b * 2^-53 is assembled from two exact int->double "magic number" conversions and one FMA
//     (a < 2^26, b < 2^27: the sum has at most 53 significant bits, so the FMA is exact) instead of I2F.F64.U64;
//   * U(0,1) skips the affine map; no bounds checks; the drain addresses are loop-invariant plus immediates.
__device__ __forceinline__ void xs_step32(uint32_t& lo, uint32_t& hi, uint32_t c21, uint32_t c4) {
    unsigned long long w = (unsigned long long)lo * c21;          // {lo >> 11, lo << 21}
    uint32_t h = hi * c21 + (uint32_t)(w >> 32);                  // hi << 21 | lo >> 11   (disjoint bits: + is |)
    hi ^= h;
    lo ^= (uint32_t)w;
    lo ^= hi >> 3;                                                // s ^= s >>> 35
    w = (unsigned long long)lo * c4;
    h = hi * c4 + (uint32_t)(w >> 32);
    hi ^= h;
    lo ^= (uint32_t)w;
}
template <bool UNIT>
__device__ __forceinline__ double xs_next_double(uint32_t& lo, uint32_t& hi, uint32_t c21, uint32_t c4, double span, double lo_) {
    xs_step32(lo, hi, c21, c4);
    const double da = __hiloint2double(0x43300000, (int)(lo & 0x3ffffffu)) - 4503599627370496.0;     // next(26), exact
    xs_step32(lo, hi, c21, c4);
    const double db = __hiloint2double(0x43300000, (int)(lo & 0x7ffffffu)) - 4503599627370496.0;     // next(27), exact
    const double x = fma(da, 0x1.0p-26, db * 0x1.0p-53);          // ((a << 27) + b) * 2^-53, exact
    return UNIT ? x : __dadd_rn(__dmul_rn(span, x), lo_);
}

template <bool UNIT>
__global__ void __launch_bounds__(256, 3) fill_uniform_fast_kernel(double* out, unsigned long long state0, long long first, double lo,
                                                               double hi, uint32_t c21, uint32_t c4) {
    __shared__ __align__(16) double stage[256][FILL_ROUND + 2];
    __shared__ unsigned long long jump_s[8][64];
    __shared__ unsigned long long base_s;
    const long long block_first = (long long)blockIdx.x * 256 * FILL_PER_THREAD;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int e = threadIdx.x; e < 8 * 64; e += 256) jump_s[e >> 6][e & 63] = g_jump[FILL_LVL0 + (e >> 6)][e & 63];
    if (warp == 0) {
        const unsigned long long b = xs_jump_warp(state0, 2ull * (unsigned long long)(first + block_first), lane);
        if (lane == 0) base_s = b;
    }
    __syncthreads();
    unsigned long long s = base_s;
#pragma unroll
    for (int j = 5; j < 8; ++j) {
        if ((warp >> (j - 5)) & 1) {
            unsigned long long v = ((s >> lane) & 1ull) ? jump_s[j][lane] : 0ull;
            v ^= ((s >> (lane + 32)) & 1ull) ? jump_s[j][lane + 32] : 0ull;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v ^= __shfl_xor_sync(0xffffffffu, v, o);
            s = v;
        }
    }
#pragma unroll 1
    for (int j = 0; j < 5; ++j) {
        if ((lane >> j) & 1) {
            unsigned long long t = 0, x = s;
            while (x) {
                t ^= jump_s[j][__ffsll((long long)x) - 1];
                x &= x - 1;
            }
            s = t;
        }
    }
    uint32_t slo = (uint32_t)s, shi = (uint32_t)(s >> 32);
    const double span = __dsub_rn(hi, lo);
    // drain: pair p = tid + 256 i of a round belongs to thread (tid >> 3) + 32 i, values 2 (tid & 7), +1: eight
    // consecutive lanes write one 128-byte line; both addresses are a per-thread constant plus i * constant
    const double* stage_rd = &stage[threadIdx.x >> 3][(threadIdx.x & 7) * 2];
    double* gdst = out + block_first + (long long)(threadIdx.x >> 3) * FILL_PER_THREAD + (threadIdx.x & 7) * 2;
#pragma unroll 1
    for (int round = 0; round < FILL_PER_THREAD / FILL_ROUND; ++round) {
#pragma unroll
        for (int v = 0; v < FILL_ROUND; v += 2) {
            double2 pr;
            pr.x = xs_next_double<UNIT>(slo, shi, c21, c4, span, lo);
            pr.y = xs_next_double<UNIT>(slo, shi, c21, c4, span, lo);
            *reinterpret_cast<double2*>(&stage[threadIdx.x][v]) = pr;
        }
        __syncthreads();
#pragma unroll
        for (int i = 0; i < FILL_ROUND / 2; ++i)
            *reinterpret_cast<double2*>(gdst + (long long)i * 32 * FILL_PER_THREAD) =
                *reinterpret_cast<const double2*>(stage_rd + i * 32 * (FILL_ROUND + 2));
        gdst += FILL_ROUND;
        __syncthreads();
    }
}

inline int ew_grid(long long work_items) {
    long long b = (work_items + EW_THREADS - 1) / EW_THREADS;
    const long long cap = 132 * 8;   // 8 resident 256-thread blocks per SM of an H100 SXM
    if (b > cap) b = cap;
    if (b < 1) b = 1;
    return (int)b;
}

}  // namespace

cudaError_t ew_binary(int op, int rows, int cols, const double* a, long long ars, long long acs, const double* b,
                      long long brs, long long bcs, double* o, long long ors, long long ocs, cudaStream_t st) {
    if (rows <= 0 || cols <= 0) return cudaSuccess;
    const long long total = (long long)rows * cols;
    const bool packed = ars == 1 && brs == 1 && ors == 1 && acs == rows && bcs == rows && ocs == rows;
    const bool aligned = ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) |
                           reinterpret_cast<uintptr_t>(o)) & 15) == 0;
    if (packed && aligned && (total % 2 == 0)) {
        const long long n2 = total / 2;
        const unsigned grid = (unsigned)((n2 + EW_THREADS * 4 - 1) / (EW_THREADS * 4));
        const double2 *a2 = reinterpret_cast<const double2*>(a), *b2 = reinterpret_cast<const double2*>(b);
        double2* o2 = reinterpret_cast<double2*>(o);
        if (op == EW_ADD) binary_flat_kernel<EW_ADD><<<grid, EW_THREADS, 0, st>>>(a2, b2, o2, n2);
        else if (op == EW_SUB) binary_flat_kernel<EW_SUB><<<grid, EW_THREADS, 0, st>>>(a2, b2, o2, n2);
        else binary_flat_kernel<EW_MUL><<<grid, EW_THREADS, 0, st>>>(a2, b2, o2, n2);
    } else {
        binary_strided_kernel<<<ew_grid(total), EW_THREADS, 0, st>>>(op, rows, cols, a, ars, acs, b, brs, bcs, o, ors, ocs);
    }
    return launched();
}

cudaError_t ew_binary_f32(int op, int rows, int cols, const float* a, long long ars, long long acs, const float* b,
                          long long brs, long long bcs, float* o, long long ors, long long ocs, cudaStream_t st) {
    if (rows <= 0 || cols <= 0) return cudaSuccess;
    binary_strided_f32_kernel<<<ew_grid((long long)rows * cols), EW_THREADS, 0, st>>>(op, rows, cols, a, ars, acs, b, brs, bcs, o,
                                                                                    ors, ocs);
    return launched();
}

cudaError_t ew_unary(int op, int rows, int cols, const double* a, long long ars, long long acs, double* o,
                     long long ors, long long ocs, double alpha, double beta, cudaStream_t st) {
    if (rows <= 0 || cols <= 0) return cudaSuccess;
    const long long total = (long long)rows * cols;
    const bool packed = ars == 1 && ors == 1 && acs == rows && ocs == rows;
    const bool aligned = ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(o)) & 15) == 0;
    if (packed && aligned && (total % 2 == 0)) {
        const long long n2 = total / 2;
        const unsigned grid = (unsigned)((n2 + EW_THREADS * 4 - 1) / (EW_THREADS * 4));
        const double2* a2 = reinterpret_cast<const double2*>(a);
        double2* o2 = reinterpret_cast<double2*>(o);
        if (op == EW_AXPB) unary_flat_kernel<EW_AXPB><<<grid, EW_THREADS, 0, st>>>(a2, o2, n2, alpha, beta);
        else if (op == EW_DIV) unary_flat_kernel<EW_DIV><<<grid, EW_THREADS, 0, st>>>(a2, o2, n2, alpha, beta);
        else if (op == EW_RDIV) unary_flat_kernel<EW_RDIV><<<grid, EW_THREADS, 0, st>>>(a2, o2, n2, alpha, beta);
        else if (op == EW_FILL) unary_flat_kernel<EW_FILL><<<grid, EW_THREADS, 0, st>>>(a2, o2, n2, alpha, beta);
        else unary_flat_kernel<EW_COPY><<<grid, EW_THREADS, 0, st>>>(a2, o2, n2, alpha, beta);
    } else {
        unary_strided_kernel<<<ew_grid(total), EW_THREADS, 0, st>>>(op, rows, cols, a, ars, acs, o, ors, ocs, alpha, beta);
    }
    return launched();
}

cudaError_t transpose_f64(const double* in, long long ldi, double* out, long long ldo, int rows, int cols,
                          cudaStream_t st) {
    if (rows <= 0 || cols <= 0) return cudaSuccess;
    const bool fast = (rows % 2 == 0) && (cols % 2 == 0) && (ldi % 2 == 0) && (ldo % 2 == 0) &&
                      (((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 15) == 0);
    if (fast) {
        const int tiles_r = (rows + TT * TT_SUB - 1) / (TT * TT_SUB), tiles_c = (cols + TT - 1) / TT;
        // 64 KiB of dynamic shared memory: above the 48 KiB a launch gets without opting in
        return launch_with_smem<transpose_f64_tile_kernel>(tiles_r * tiles_c, 256, TT_SMEM, st, in, ldi, out, ldo, rows, cols,
                                                           tiles_r, tiles_c);
    }
    dim3 grid((rows + 31) / 32, (cols + 31) / 32);
    transpose_generic_kernel<double><<<grid, 256, 0, st>>>(in, ldi, out, ldo, rows, cols);
    return launched();
}

cudaError_t transpose_b16(const void* in, long long ldi, void* out, long long ldo, int rows, int cols, cudaStream_t st) {
    if (rows <= 0 || cols <= 0) return cudaSuccess;
    dim3 grid((rows + 31) / 32, (cols + 31) / 32);
    transpose_generic_kernel<unsigned short><<<grid, 256, 0, st>>>(static_cast<const unsigned short*>(in), ldi,
                                                                  static_cast<unsigned short*>(out), ldo, rows, cols);
    return launched();
}
cudaError_t transpose_b32(const void* in, long long ldi, void* out, long long ldo, int rows, int cols, cudaStream_t st) {
    if (rows <= 0 || cols <= 0) return cudaSuccess;
    dim3 grid((rows + 31) / 32, (cols + 31) / 32);
    transpose_generic_kernel<unsigned int><<<grid, 256, 0, st>>>(static_cast<const unsigned int*>(in), ldi,
                                                                static_cast<unsigned int*>(out), ldo, rows, cols);
    return launched();
}

int sum_scratch_doubles() { return SUM_BLOCKS + 1; }

cudaError_t sum_f64(const double* a, int rows, int cols, long long ld, double* scratch, cudaStream_t st) {
    // scratch[0] receives the result, scratch[1..] the per-block partials
    const long long total = (long long)rows * cols;
    int blocks = (int)min((long long)SUM_BLOCKS, max(1ll, (total + 2047) / 2048));      // one CTA per 16 KiB tile, capped
    sum_strided_kernel<<<blocks, 256, 0, st>>>(a, rows, cols, ld, scratch + 1);
    if (const cudaError_t e = launched(); e != cudaSuccess) return e;
    sum_final_kernel<<<1, 256, 0, st>>>(scratch + 1, blocks, scratch);
    return launched();
}

template <typename TI, typename TO>
static cudaError_t convert_t(int rows, int cols, const void* a, long long ars, long long acs, void* o, long long ors,
                             long long ocs, cudaStream_t st) {
    if (rows <= 0 || cols <= 0) return cudaSuccess;
    convert_strided_kernel<TI, TO><<<ew_grid((long long)rows * cols), EW_THREADS, 0, st>>>(
        rows, cols, static_cast<const TI*>(a), ars, acs, static_cast<TO*>(o), ors, ocs);
    return launched();
}

// dtype codes follow mb_dtype: 0 = f64, 1 = bf16, 2 = f32
cudaError_t convert_strided(int src_dtype, int dst_dtype, int rows, int cols, const void* a, long long ars,
                            long long acs, void* o, long long ors, long long ocs, cudaStream_t st) {
    using bf = __nv_bfloat16;
    if (src_dtype == 0 && dst_dtype == 0) return convert_t<double, double>(rows, cols, a, ars, acs, o, ors, ocs, st);
    if (src_dtype == 0 && dst_dtype == 1) return convert_t<double, bf>(rows, cols, a, ars, acs, o, ors, ocs, st);
    if (src_dtype == 0 && dst_dtype == 2) return convert_t<double, float>(rows, cols, a, ars, acs, o, ors, ocs, st);
    if (src_dtype == 1 && dst_dtype == 0) return convert_t<bf, double>(rows, cols, a, ars, acs, o, ors, ocs, st);
    if (src_dtype == 2 && dst_dtype == 0) return convert_t<float, double>(rows, cols, a, ars, acs, o, ors, ocs, st);
    if (src_dtype == 1 && dst_dtype == 1) return convert_t<bf, bf>(rows, cols, a, ars, acs, o, ors, ocs, st);
    if (src_dtype == 2 && dst_dtype == 2) return convert_t<float, float>(rows, cols, a, ars, acs, o, ors, ocs, st);
    if (src_dtype == 1 && dst_dtype == 2) return convert_t<bf, float>(rows, cols, a, ars, acs, o, ors, ocs, st);
    if (src_dtype == 2 && dst_dtype == 1) return convert_t<float, bf>(rows, cols, a, ars, acs, o, ors, ocs, st);
    return cudaErrorInvalidValue;
}

// ---- XORShift jump tables (host) ----
static unsigned long long h_step(unsigned long long s) {
    s ^= s << 21;
    s ^= s >> 35;
    s ^= s << 4;
    return s;
}
cudaError_t fill_uniform_init_tables() {
    static std::mutex mu;                      // first calls from several host threads serialise here
    static std::atomic<bool> done[64];
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev >= 0 && dev < 64 && done[dev].load(std::memory_order_acquire)) return cudaSuccess;
    std::lock_guard<std::mutex> lk(mu);
    static unsigned long long tab[40][64];
    static bool built = false;
    if (!built) {
        // column b of T^1 = step(1<<b); T^(2^(j+1)) = T^(2^j) applied to the columns of T^(2^j)
        for (int b = 0; b < 64; ++b) tab[0][b] = h_step(1ull << b);
        for (int j = 1; j < 40; ++j) {
            for (int b = 0; b < 64; ++b) {
                unsigned long long x = tab[j - 1][b], t = 0;
                for (int c = 0; c < 64; ++c)
                    if ((x >> c) & 1ull) t ^= tab[j - 1][c];
                tab[j][b] = t;
            }
        }
        built = true;
    }
    cudaError_t e = cudaMemcpyToSymbol(g_jump, tab, sizeof(tab));
    if (e == cudaSuccess && dev >= 0 && dev < 64) done[dev].store(true, std::memory_order_release);
    return e;
}

cudaError_t fill_jump_tables(const unsigned long long** tables) {
    cudaError_t e = fill_uniform_init_tables();
    if (e != cudaSuccess) return e;
    void* p = nullptr;
    e = cudaGetSymbolAddress(&p, g_jump);
    *tables = static_cast<const unsigned long long*>(p);
    return e;
}

// The fast kernel must reproduce the general kernel (the one pinned against the JVM stream) bit for bit.  That is checked
// ONCE per device and process, on the device itself: two CTAs of each kernel at a far, odd stream offset, unit and affine
// range, compared on the host (about a millisecond).  A mismatch — a compiler or driver that breaks one of the kernel's
// exactness arguments — disables the fast kernel for the process and says so on stderr; results stay those of the general
// kernel either way.  Returns 1 (verified) or -1 (disabled).  Its launches are not counted (no launched()): they are not
// the work of the call that happens to run the check.
static int fast_fill_state(cudaStream_t st) {
    static std::mutex mu;
    static std::atomic<int> state[64];
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) return -1;
    int s = state[dev].load(std::memory_order_acquire);
    if (s) return s;
    std::lock_guard<std::mutex> lk(mu);
    s = state[dev].load(std::memory_order_acquire);
    if (s) return s;
    const long long n = 2 * 256ll * FILL_PER_THREAD;
    const unsigned long long st0 = 0x9E3779B97F4A7C15ull;
    const long long first = (1ll << 35) + 12345;
    double* d = nullptr;
    bool ok = cudaMalloc(&d, 2 * n * sizeof(double)) == cudaSuccess;
    std::vector<double> h(ok ? 2 * n : 0);
    for (int variant = 0; variant < 2 && ok; ++variant) {
        const double lo = variant ? -2.0 : 0.0, hi = variant ? 5.0 : 1.0;
        fill_uniform_kernel<<<2, 256, 0, st>>>(d, 1, n, (int)n, 1, 0, st0, first, lo, hi, 0);
        if (variant)
            fill_uniform_fast_kernel<false><<<2, 256, 0, st>>>(d + n, st0, first, lo, hi, 1u << 21, 1u << 4);
        else
            fill_uniform_fast_kernel<true><<<2, 256, 0, st>>>(d + n, st0, first, lo, hi, 1u << 21, 1u << 4);
        ok = cudaGetLastError() == cudaSuccess &&
             cudaMemcpyAsync(h.data(), d, 2 * n * sizeof(double), cudaMemcpyDeviceToHost, st) == cudaSuccess &&
             cudaStreamSynchronize(st) == cudaSuccess && memcmp(h.data(), h.data() + n, n * sizeof(double)) == 0;
    }
    if (d) cudaFree(d);
    if (!ok)
        fprintf(stderr, "marlin_b200: the fast generator kernel does not reproduce the reference-exact kernel on device %d; "
                        "it is disabled for this process (mb_fill_uniform keeps using the general kernel)\n", dev);
    s = ok ? 1 : -1;
    state[dev].store(s, std::memory_order_release);
    return s;
}

cudaError_t fill_uniform_f64(double* out, long long rs, long long cs, int rows, int cols, int row_major,
                             unsigned long long state0, long long first, double lo, double hi, cudaStream_t st) {
    if (rows <= 0 || cols <= 0) return cudaSuccess;
    cudaError_t e = fill_uniform_init_tables();
    if (e != cudaSuccess) return e;
    const long long total = (long long)rows * cols;
    const long long per_block = 256ll * FILL_PER_THREAD;
    const int blocks = (int)((total + per_block - 1) / per_block);
    // full CTAs of a linear, 16-byte aligned destination take the fast kernel; the ragged last CTA and strided
    // destinations the general one
    const bool linear = row_major ? (cs == 1 && rs == cols) : (rs == 1 && cs == rows);
    int full = 0;
    if (linear &&((reinterpret_cast<uintptr_t>(out) & 15) == 0) && total >= per_block && fast_fill_state(st) > 0)
        full = (int)(total / per_block);
    if (full > 0) {
        if (lo == 0.0 && hi == 1.0)
            fill_uniform_fast_kernel<true><<<full, 256, 0, st>>>(out, state0, first, lo, hi, 1u << 21, 1u << 4);
        else
            fill_uniform_fast_kernel<false><<<full, 256, 0, st>>>(out, state0, first, lo, hi, 1u << 21, 1u << 4);
        if ((e = launched()) != cudaSuccess) return e;
    }
    if (blocks == full) return cudaSuccess;
    fill_uniform_kernel<<<blocks - full, 256, 0, st>>>(out, rs, cs, rows, cols, row_major, state0, first, lo, hi, full);
    return launched();
}

}  // namespace mb

// StandardNormalGenerator(mean, variance).nextValue() (utils/RandomDataGenerator.scala:70-82) for a whole partition,
// bit-exact with the JVM: value k is mean + sqrt(variance) * g_k, g the output of java.util.Random.nextGaussian running
// over XORShiftRandom.next (:113-131).  nextGaussian is the polar method: attempt a takes nextDouble positions 2a and 2a+1
// (XORShift steps 4a+1 .. 4a+4), v = 2u - 1, s = v1^2 + v2^2, rejects s >= 1 and s == 0, and turns an accepted attempt
// into the pair v1 * m, v2 * m with m = sqrt(-2 log(s) / s) (StrictMath: fdlibm's log).
//
// Where value k lands depends on how many earlier attempts were rejected, so the XORShift jump-ahead alone cannot place
// it.  Three passes, none of which waits on another CTA:
//   count  the attempts are cut into tiles of NORMAL_TILE_ATTEMPTS; thread t of the tile's CTA jumps to its run of
//          NORMAL_RUN attempts and counts the accepted ones (integer work, two exact DADDs, two DMULs and one DADD per
//          attempt, no log).  The CTA stores the tile's count and every thread's exclusive prefix within the tile.
//   scan   one CTA turns the tile counts into exclusive prefixes (and their total) in pairs.
//   write  the CTA of tile t regenerates its attempts; accepted attempt r of the tile becomes values 2 (prefix_t + r) and
//          2 (prefix_t + r) + 1, clipped at n, so the tile's output is one contiguous range of fill order.  It goes out
//          through shared memory in rounds, as fill_uniform_kernel's does.
// The host counts a first budget of tiles and further rounds while the total falls short (see MB_NORMAL_TILE_ATTEMPTS).
//
// Every operation of the polar step, the log and the scaling is an explicit __dmul_rn / __dadd_rn / __dsub_rn, so nothing
// contracts into an FMA; the divisions and the square root are correctly rounded and live in out-of-line functions
// (div_rn, polar_multiplier), whose DFMA sequences are the only ones in the write kernel.
#include "normal.h"
#include "elementwise.h"
#include "launch.h"
#include "stream_buffer.h"

#include <cmath>
#include <cstdint>

namespace mb {
namespace {

constexpr int NORMAL_THREADS = 256;
constexpr int NORMAL_RUN = NORMAL_TILE_ATTEMPTS / NORMAL_THREADS;      // 128 attempts per thread
constexpr int NORMAL_ROUND = 8;                                        // attempts per thread between two stage drains
constexpr int NORMAL_LVL0 = 9;          // thread offset = t * 4 * NORMAL_RUN steps = t << 9: table levels 9..16
constexpr int NORMAL_TILE_LOG2_STEPS = 17;                             // 4 * NORMAL_TILE_ATTEMPTS = 2^17 steps per tile
static_assert(4 * NORMAL_RUN == 1 << NORMAL_LVL0, "thread runs must start on a jump-table level");
static_assert(4ll * NORMAL_TILE_ATTEMPTS == 1ll << NORMAL_TILE_LOG2_STEPS, "tiles must start on a jump-table level");

__device__ __forceinline__ unsigned long long xs_step(unsigned long long s) {
    s ^= s << 21;
    s ^= s >> 35;
    s ^= s << 4;
    return s;
}

// 2^52 v for the stream's next nextDouble u, v = 2u - 1 = (x - 2^52) 2^-52 with x = next(26) << 27 | next(27) (exact).
// |x - 2^52| is placed in the significand of +-(2^52 + |x - 2^52|) and one exact DADD takes the 2^52 off again; at
// x = 0 the carry into the exponent still gives the right value, -2^53.
__device__ __forceinline__ double next_v52(unsigned long long& s) {
    s = xs_step(s);
    const unsigned long long hi26 = s & ((1ull << 26) - 1);
    s = xs_step(s);
    const unsigned long long lo27 = s & ((1ull << 27) - 1);
    const long long t = (long long)((hi26 << 27) | lo27) - (1ll << 52);
    const bool neg = t < 0;
    const unsigned long long mag = neg ? (unsigned long long)(-t) : (unsigned long long)t;
    const double d = __longlong_as_double((long long)((neg ? 0xC330000000000000ull : 0x4330000000000000ull) + mag));
    return __dadd_rn(d, neg ? 0x1p52 : -0x1p52);
}

// The attempt's s scaled by 2^104: fl(fl(T1^2) + fl(T2^2)) with T = 2^52 v is exactly 2^104 fl(fl(v1^2) + fl(v2^2)),
// because v^2 >= 2^-104 never underflows.  So the JVM's test s < 1 && s != 0 is q < 2^104 && q != 0.
__device__ __forceinline__ double attempt_q(double t1, double t2) { return __dadd_rn(__dmul_rn(t1, t1), __dmul_rn(t2, t2)); }
__device__ __forceinline__ bool accepted(double q) { return q < 0x1p104 && q != 0.0; }

// Correctly rounded division, out of line (see polar_multiplier).
__device__ __noinline__ double div_rn(double a, double b) { return __ddiv_rn(a, b); }

// java.lang.StrictMath.log (fdlibm e_log.c) for positive normal x < 1, the only inputs nextGaussian gives it; the same
// operations in the same order as hostlogic.cpp's fdlibm_log.
__device__ __forceinline__ double fdlibm_log(double x) {
    const double ln2_hi = 6.93147180369123816490e-01, ln2_lo = 1.90821492927058770002e-10;
    const double Lg1 = 6.666666666666735130e-01, Lg2 = 3.999999999940941908e-01, Lg3 = 2.857142874366239149e-01,
                 Lg4 = 2.222219843214978396e-01, Lg5 = 1.818357216161805012e-01, Lg6 = 1.531383769920937332e-01,
                 Lg7 = 1.479819860511658591e-01;
    const long long bits = __double_as_longlong(x);
    int hx = (int)(bits >> 32);
    int k = (hx >> 20) - 1023;
    hx &= 0x000fffff;
    int i = (hx + 0x95f64) & 0x100000;
    x = __longlong_as_double(((long long)(hx | (i ^ 0x3ff00000)) << 32) | (bits & 0xffffffffll));     // x or x / 2
    k += i >> 20;
    const double f = __dsub_rn(x, 1.0), dk = (double)k;
    if ((0x000fffff & (2 + hx)) < 3) {                                                                  // |f| < 2^-20
        if (f == 0.0) return k == 0 ? 0.0 : __dadd_rn(__dmul_rn(dk, ln2_hi), __dmul_rn(dk, ln2_lo));
        const double R = __dmul_rn(__dmul_rn(f, f), __dsub_rn(0.5, __dmul_rn(0.33333333333333333, f)));
        return k == 0 ? __dsub_rn(f, R) : __dsub_rn(__dmul_rn(dk, ln2_hi), __dsub_rn(__dsub_rn(R, __dmul_rn(dk, ln2_lo)), f));
    }
    const double s = div_rn(f, __dadd_rn(2.0, f));
    const double z = __dmul_rn(s, s), w = __dmul_rn(z, z);
    i = hx - 0x6147a;
    const int j = 0x6b851 - hx;
    const double t1 = __dmul_rn(w, __dadd_rn(Lg2, __dmul_rn(w, __dadd_rn(Lg4, __dmul_rn(w, Lg6)))));
    const double t2 = __dmul_rn(z, __dadd_rn(Lg1, __dmul_rn(w, __dadd_rn(Lg3, __dmul_rn(w, __dadd_rn(Lg5, __dmul_rn(w, Lg7)))))));
    i |= j;
    const double R = __dadd_rn(t2, t1);
    if (i > 0) {
        const double hfsq = __dmul_rn(__dmul_rn(0.5, f), f);
        const double sh = __dmul_rn(s, __dadd_rn(hfsq, R));
        return k == 0 ? __dsub_rn(f, __dsub_rn(hfsq, sh))
                      : __dsub_rn(__dmul_rn(dk, ln2_hi), __dsub_rn(__dsub_rn(hfsq, __dadd_rn(sh, __dmul_rn(dk, ln2_lo))), f));
    }
    const double sf = __dmul_rn(s, __dsub_rn(f, R));
    return k == 0 ? __dsub_rn(f, sf) : __dsub_rn(__dmul_rn(dk, ln2_hi), __dsub_rn(__dsub_rn(sf, __dmul_rn(dk, ln2_lo)), f));
}

// StrictMath.sqrt(-2 * log(s) / s) from -2 log(s): both roundings correct.  Out of line like div_rn, so the DFMA sequences
// of the divisions and the square root stay apart from the kernel bodies (tests/test_sass_normal.py).
__device__ __noinline__ double polar_multiplier(double minus2log, double s) { return __dsqrt_rn(__ddiv_rn(minus2log, s)); }

// The XORShift state before attempt tile * NORMAL_TILE_ATTEMPTS + threadIdx.x * NORMAL_RUN: warp 0 jumps to the tile
// (whole-warp matrix products from the global tables), then three warp-cooperative levels for the warp's part of the
// offset and five serial ones for the lane's, from levels NORMAL_LVL0 .. +7 staged in shared memory (fill_uniform_kernel's
// scheme).  Every thread of the CTA calls it.
__device__ __forceinline__ unsigned long long run_start(unsigned long long state0, const unsigned long long* __restrict__ tab,
                                                        long long tile, unsigned long long (*jump_s)[64],
                                                        unsigned long long* base_s) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int e = threadIdx.x; e < 8 * 64; e += NORMAL_THREADS) jump_s[e >> 6][e & 63] = tab[(NORMAL_LVL0 + (e >> 6)) * 64 + (e & 63)];
    if (warp == 0) {
        unsigned long long s = state0;
        unsigned long long steps = (unsigned long long)tile;
        for (int j = NORMAL_TILE_LOG2_STEPS; j < 40 && steps; ++j, steps >>= 1) {
            if (steps & 1ull) {
                unsigned long long v = ((s >> lane) & 1ull) ? tab[j * 64 + lane] : 0ull;
                v ^= ((s >> (lane + 32)) & 1ull) ? tab[j * 64 + lane + 32] : 0ull;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) v ^= __shfl_xor_sync(0xffffffffu, v, o);
                s = v;
            }
        }
        if (lane == 0) *base_s = s;
    }
    __syncthreads();
    unsigned long long s = *base_s;
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
    return s;
}

// Tiles tile0 .. tile0 + gridDim.x - 1: tile_cnt[tile] = its accepted attempts, thr_pre[tile * 256 + t] = those of the
// runs before thread t's.
__global__ void __launch_bounds__(NORMAL_THREADS) normal_count_kernel(unsigned long long state0, const unsigned long long* __restrict__ tab,
                                                                    long long tile0, int* __restrict__ tile_cnt,
                                                                    uint16_t* __restrict__ thr_pre) {
    __shared__ unsigned long long jump_s[8][64];
    __shared__ unsigned long long base_s;
    __shared__ int warp_s[NORMAL_THREADS / 32];
    const long long tile = tile0 + blockIdx.x;
    unsigned long long s = run_start(state0, tab, tile, jump_s, &base_s);
    int c = 0;
#pragma unroll 4
    for (int a = 0; a < NORMAL_RUN; ++a) {
        const double t1 = next_v52(s);
        const double t2 = next_v52(s);
        c += accepted(attempt_q(t1, t2)) ? 1 : 0;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    if (lane == 31) warp_s[warp] = incl;
    __syncthreads();
    int before = 0, total = 0;
#pragma unroll
    for (int w = 0; w < NORMAL_THREADS / 32; ++w) {
        before += w < warp ? warp_s[w] : 0;
        total += warp_s[w];
    }
    thr_pre[tile * NORMAL_THREADS + threadIdx.x] = (uint16_t)(before + incl - c);
    if (threadIdx.x == 0) tile_cnt[tile] = total;
}

// pre[t] = sum of cnt[0 .. t), pre[len] = the total.
__global__ void __launch_bounds__(1024) normal_scan_kernel(const int* __restrict__ cnt, long long len, long long* __restrict__ pre) {
    __shared__ long long part[1024];
    const long long per = (len + 1023) / 1024;
    const long long b = threadIdx.x * per, e = min(len, b + per);
    long long s = 0;
    for (long long i = b; i < e; ++i) s += cnt[i];
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
        pre[i] = run;
        run += cnt[i];
    }
    if (threadIdx.x == 1023) pre[len] = run;
}

// Tile blockIdx.x: the pairs from pre[tile] on, as far as value n - 1.  Each thread regenerates its run in rounds of
// NORMAL_ROUND attempts; a round's accepted pairs of thread t sit in stage[t] and belong at pair dst_s[t] onwards, a
// contiguous piece of fill order, which the whole CTA then stores.  *attempts_used = A from the thread that produces pair
// ceil(n / 2) - 1.
__global__ void __launch_bounds__(NORMAL_THREADS) normal_write_kernel(double* __restrict__ out, long long rs, long long cs, int rows,
                                                                    int cols, int row_major, unsigned long long state0,
                                                                    const unsigned long long* __restrict__ tab,
                                                                    const long long* __restrict__ pre,
                                                                    const uint16_t* __restrict__ thr_pre, double mean, double sd,
                                                                    long long* __restrict__ attempts_used) {
    __shared__ __align__(16) double stage[NORMAL_THREADS][2 * NORMAL_ROUND + 2];     // 16-byte rows, conflict-free pairs
    __shared__ unsigned long long jump_s[8][64];
    __shared__ unsigned long long base_s;
    __shared__ long long dst_s[NORMAL_THREADS];
    __shared__ int cnt_s[NORMAL_THREADS];
    const long long n = (long long)rows * cols, pairs = (n + 1) / 2;
    const long long tile = blockIdx.x;
    const long long tile_first = pre[tile];
    if (tile_first >= pairs) return;                                   // the whole CTA: a tile past the last pair
    unsigned long long s = run_start(state0, tab, tile, jump_s, &base_s);
    long long next = tile_first + thr_pre[tile * NORMAL_THREADS + threadIdx.x];
    long long attempt = tile * NORMAL_TILE_ATTEMPTS + (long long)threadIdx.x * NORMAL_RUN;
    const bool linear = row_major ? (cs == 1 && rs == cols) : (rs == 1 && cs == rows);
    const bool vec = linear && ((reinterpret_cast<uintptr_t>(out) & 15) == 0);
#pragma unroll 1
    for (int round = 0; round < NORMAL_RUN / NORMAL_ROUND; ++round) {
        const bool active = next < pairs;
        if (!__syncthreads_or(active)) break;
        int cnt = 0;
        if (active) {
#pragma unroll 1
            for (int i = 0; i < NORMAL_ROUND; ++i) {
                const double t1 = next_v52(s);
                const double t2 = next_v52(s);
                const double q = attempt_q(t1, t2);
                if (accepted(q)) {
                    const double sv = __dmul_rn(q, 0x1p-104);                                 // exact
                    const double m = polar_multiplier(__dmul_rn(-2.0, fdlibm_log(sv)), sv);
                    double2 v;
                    v.x = __dadd_rn(mean, __dmul_rn(sd, __dmul_rn(__dmul_rn(t1, 0x1p-52), m)));
                    v.y = __dadd_rn(mean, __dmul_rn(sd, __dmul_rn(__dmul_rn(t2, 0x1p-52), m)));
                    *reinterpret_cast<double2*>(&stage[threadIdx.x][2 * cnt]) = v;
                    if (next + cnt == pairs - 1 && attempts_used) *attempts_used = attempt + i + 1;
                    ++cnt;
                }
            }
        }
        dst_s[threadIdx.x] = next;
        cnt_s[threadIdx.x] = cnt;
        next += cnt;
        attempt += NORMAL_ROUND;
        __syncthreads();
        if (vec) {
            // pair j of owner thread o: e = o * NORMAL_ROUND + j, eight lanes per owner, one 16-byte store each
#pragma unroll
            for (int e = threadIdx.x; e < NORMAL_THREADS * NORMAL_ROUND; e += NORMAL_THREADS) {
                const int o = e / NORMAL_ROUND, j = e % NORMAL_ROUND;
                if (j < cnt_s[o]) {
                    const long long idx = 2 * (dst_s[o] + j);
                    if (idx + 1 < n) *reinterpret_cast<double2*>(out + idx) = *reinterpret_cast<const double2*>(&stage[o][2 * j]);
                    else if (idx < n) out[idx] = stage[o][2 * j];
                }
            }
        } else {
#pragma unroll 4
            for (int e = threadIdx.x; e < NORMAL_THREADS * 2 * NORMAL_ROUND; e += NORMAL_THREADS) {
                const int o = e / (2 * NORMAL_ROUND), j = e % (2 * NORMAL_ROUND);
                if (j < 2 * cnt_s[o]) {
                    const long long i = 2 * dst_s[o] + j;
                    if (i < n) {
                        if (linear) {
                            out[i] = stage[o][j];
                        } else {
                            long long r, c;
                            if (row_major) { r = i / cols; c = i - r * cols; } else { c = i / rows; r = i - c * rows; }
                            out[r * rs + c * cs] = stage[o][j];
                        }
                    }
                }
            }
        }
    }
}

// Tiles counted for a deficit of `pairs` pairs: ceil(ceil(pairs * 4 / pi) / NORMAL_TILE_ATTEMPTS) (MB_NORMAL_TILE_ATTEMPTS).
long long budget_tiles(long long pairs) {
    const long long attempts = (long long)std::ceil((double)pairs * 4.0 / 3.141592653589793);
    return (attempts + NORMAL_TILE_ATTEMPTS - 1) / NORMAL_TILE_ATTEMPTS;
}

// The per-call arrays of `cap` tiles in one allocation: pre[cap + 1], attempts_used, cnt[cap], thr_pre[cap * 256].
struct TileArrays {
    StreamBuffer buf;
    long long cap = 0;
    long long* pre() const { return buf.as<long long>(); }
    long long* used() const { return buf.as<long long>() + cap + 1; }
    int* cnt() const { return reinterpret_cast<int*>(used() + 1); }
    uint16_t* thr() const { return reinterpret_cast<uint16_t*>(cnt() + cap); }
    static size_t bytes(long long cap) { return (size_t)(cap + 2) * 8 + (size_t)cap * 4 + (size_t)cap * NORMAL_THREADS * 2; }
    cudaError_t alloc(long long c, cudaStream_t st) {
        cap = c;
        return buf.alloc(bytes(c), st);
    }
};

}  // namespace

cudaError_t fill_normal_f64(double* out, long long rs, long long cs, int rows, int cols, int row_major,
                            unsigned long long state0, double mean, double sd, long long max_positions,
                            long long* attempts_used, cudaStream_t st) {
    if (attempts_used) *attempts_used = 0;
    if (rows <= 0 || cols <= 0) return cudaSuccess;
    const unsigned long long* tab = nullptr;
    cudaError_t e = fill_jump_tables(&tab);
    if (e != cudaSuccess) return e;
    const long long pairs = ((long long)rows * cols + 1) / 2;
    // two allocations take turns when a further round needs room: the counts so far are copied over
    TileArrays arr[2];
    int cur = 0;
    long long counted = 0, add = budget_tiles(pairs), total = 0;
    for (;;) {
        if (2 * (counted + add) * NORMAL_TILE_ATTEMPTS > max_positions) return cudaErrorInvalidValue;
        if (counted + add > arr[cur].cap) {
            TileArrays& nx = arr[1 - cur];
            if ((e = nx.alloc(counted + add, st)) != cudaSuccess) return e;
            if (counted) {
                e = cudaMemcpyAsync(nx.cnt(), arr[cur].cnt(), sizeof(int) * counted, cudaMemcpyDeviceToDevice, st);
                if (e == cudaSuccess)
                    e = cudaMemcpyAsync(nx.thr(), arr[cur].thr(), sizeof(uint16_t) * NORMAL_THREADS * counted,
                                        cudaMemcpyDeviceToDevice, st);
                if (e != cudaSuccess) return e;
            }
            cur = 1 - cur;
        }
        const TileArrays& a = arr[cur];
        normal_count_kernel<<<(unsigned)add, NORMAL_THREADS, 0, st>>>(state0, tab, counted, a.cnt(), a.thr());
        if ((e = launched()) != cudaSuccess) return e;
        counted += add;
        normal_scan_kernel<<<1, 1024, 0, st>>>(a.cnt(), counted, a.pre());
        if ((e = launched()) != cudaSuccess) return e;
        if ((e = cudaMemcpyAsync(&total, a.pre() + counted, sizeof(long long), cudaMemcpyDeviceToHost, st)) != cudaSuccess) return e;
        if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return e;
        if (total >= pairs) break;
        add = budget_tiles(pairs - total);
    }
    const TileArrays& a = arr[cur];
    normal_write_kernel<<<(unsigned)counted, NORMAL_THREADS, 0, st>>>(out, rs, cs, rows, cols, row_major, state0, tab, a.pre(),
                                                                      a.thr(), mean, sd, attempts_used ? a.used() : nullptr);
    if ((e = launched()) != cudaSuccess) return e;
    if (!attempts_used) return cudaSuccess;
    if ((e = cudaMemcpyAsync(attempts_used, a.used(), sizeof(long long), cudaMemcpyDeviceToHost, st)) != cudaSuccess) return e;
    return cudaStreamSynchronize(st);
}

}  // namespace mb

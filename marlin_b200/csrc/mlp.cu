// The NeuralNetwork example (examples/NeuralNetwork.scala) between its two large GEMMs: see mlp.h for the arithmetic.
//
// nn_backprop_kernel: a persistent CTA owns tiles of NN_ROWS rows of one block's Z1 (tiles blockIdx.x, blockIdx.x +
// gridDim.x, ...).  Warp 0 streams a tile in pieces of NN_CHUNK columns into a shared-memory ring with plain bulk copies
// (one cp.async.bulk per column, completing on the stage's mbarrier), so any ld and any 8-byte alignment is read in place.
//   pass A  warp w, lane = row: columns w, w + 8, ... of each piece become A1 = sigmoid(Z1) where they landed and add into
//           the lane's ten partial sums of Z2; the eight warps' partials are summed in warp order, and D2 is formed.
//   pass B  the same mapping: E1 = D2 W2^T from the lane's row of D2, D1 = (1 - A1) A1 E1 stored to the output; then, four
//           threads per column, A1^T D2 adds into the CTA's partial over the tile's rows in ascending order.
// For H <= NN_RESIDENT_H the whole tile stays in the ring between the passes, the output weight sits in shared memory as
// rows of ten, and the next tile streams in while pass B frees the stages: Z1 crosses HBM once.  Wider layers stream each
// piece a second time for pass B (the sigmoid is evaluated again by the same function, so A1 is the same bits) and read
// the output weight through the read-only cache.
// A1, Z2, A2 and D2 exist only in shared memory and registers.  No atomics: the same inputs give the same bits.
#include "mlp.h"
#include "ptx.cuh"
#include "launch.h"

#include <cstdint>

namespace mb {
namespace {

constexpr int NN_ROWS = 32;                  // rows per tile: one per lane
constexpr int NN_THREADS = 256;
constexpr int NN_WARPS = NN_THREADS / 32;
constexpr int NN_CHUNK = 64;                 // columns per piece
constexpr int NN_SLOT = NN_ROWS + 2;         // doubles per column slot: the rows plus a 16-byte alignment lead and tail
constexpr int NN_STAGES = NN_RESIDENT_H / NN_CHUNK;
constexpr int NN_STAGE_DOUBLES = NN_CHUNK * NN_SLOT;
constexpr int NN_SMEM_DOUBLES = NN_STAGES * NN_STAGE_DOUBLES + NN_RESIDENT_H * NN_CLASSES + NN_WARPS * NN_ROWS * NN_CLASSES +
                                NN_ROWS * NN_CLASSES + NN_STAGES;
constexpr int NN_SMEM = NN_SMEM_DOUBLES * 8;
static_assert(NN_CLASSES == 10, "the kernel's thread mappings are written for ten output units");

struct NnShape {
    const double* z;
    long long ld;
    int r, H;
    int nch;          // pieces per tile
    int per_tile;     // loads per tile: nch, or 2 * nch when pass B streams the tile again
    int ntiles;
};

// sigmoid(x) = 1 / (1 + exp(-x)) with IEEE division (breeze.numerics.sigmoid), the form of logistic.cu's gradientMul.  Out
// of line so that both passes call the same instructions.
__device__ __noinline__ double nn_sigmoid(double x) { return __ddiv_rn(1.0, __dadd_rn(1.0, exp(-x))); }

// Warp 0 (all lanes): issue load k of this CTA's sequence into stage k % NN_STAGES, if it exists.
__device__ __forceinline__ void nn_issue(const NnShape& s, int k, double* ring, uint64_t* full) {
    const int q = k / s.per_tile;
    const int c = (k % s.per_tile) % s.nch;
    const long long t = blockIdx.x + (long long)q * gridDim.x;
    if (t >= s.ntiles) return;
    const int lane = threadIdx.x & 31;
    const long long r0 = t * NN_ROWS;
    const int nr = static_cast<int>(min((long long)NN_ROWS, s.r - r0));
    const int c0 = c * NN_CHUNK, cw = min(NN_CHUNK, s.H - c0);
    const int stage = k % NN_STAGES;
    uint32_t bytes[NN_CHUNK / 32] = {};
    const double* src[NN_CHUNK / 32] = {};
    uint32_t mine = 0;
#pragma unroll
    for (int i = 0; i < NN_CHUNK / 32; ++i) {
        const int hh = lane + 32 * i;
        int lead = 0;
        if (hh < cw) src[i] = piece_span(s.z + r0 + (c0 + hh) * s.ld, nr, &bytes[i], &lead);
        mine += bytes[i];
    }
    const uint32_t total = __reduce_add_sync(0xffffffffu, mine);
    const uint32_t bar = smem_u32(&full[stage]);
    if (lane == 0) mbar_arrive_expect_tx(bar, total);
    __syncwarp();
#pragma unroll
    for (int i = 0; i < NN_CHUNK / 32; ++i)
        if (bytes[i]) bulk_load(smem_u32(ring + (long long)stage * NN_STAGE_DOUBLES + (lane + 32 * i) * NN_SLOT), src[i], bytes[i], bar);
}

__device__ __forceinline__ void nn_wait(const uint64_t* full, int k) {
    mbar_wait(smem_u32(&full[k % NN_STAGES]), static_cast<uint32_t>((k / NN_STAGES) & 1));
}

// Row h of the output weight: from its shared-memory copy (rows of ten) or, for a wide layer, from the column-major array.
__device__ __forceinline__ void nn_w2_row(double (&w)[NN_CLASSES], const double* w2s, const double* __restrict__ w2, long long ldw2,
                                          int h, bool resident) {
    if (resident) {
        const double2* p = reinterpret_cast<const double2*>(w2s + h * NN_CLASSES);
#pragma unroll
        for (int j = 0; j < NN_CLASSES / 2; ++j) {
            const double2 v = p[j];
            w[2 * j] = v.x;
            w[2 * j + 1] = v.y;
        }
    } else {
#pragma unroll
        for (int j = 0; j < NN_CLASSES; ++j) w[j] = __ldg(w2 + h + j * ldw2);
    }
}

__global__ void __launch_bounds__(NN_THREADS, 1)
nn_backprop_kernel(NnShape s, const double* __restrict__ w2, long long ldw2, const int* __restrict__ labels, double* d1,
                   long long ldd, double* part) {
    extern __shared__ __align__(16) unsigned char nn_smem[];
    double* ring = reinterpret_cast<double*>(nn_smem);
    double* w2s = ring + NN_STAGES * NN_STAGE_DOUBLES;
    double* zs = w2s + NN_RESIDENT_H * NN_CLASSES;          // [warp][row][class]: the warps' partial sums of Z2
    double* d2s = zs + NN_WARPS * NN_ROWS * NN_CLASSES;      // [row][class]
    uint64_t* full = reinterpret_cast<uint64_t*>(d2s + NN_ROWS * NN_CLASSES);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int H = s.H;
    const bool resident = s.per_tile == s.nch;
    double* mypart = part + (long long)blockIdx.x * H * NN_CLASSES;
    for (int i = tid; i < H * NN_CLASSES; i += NN_THREADS) mypart[i] = 0.0;
    if (resident)
        for (int i = tid; i < H * NN_CLASSES; i += NN_THREADS) w2s[i] = w2[i / NN_CLASSES + (i % NN_CLASSES) * ldw2];
    if (tid == 0) {
        for (int i = 0; i < NN_STAGES; ++i) mbar_init(smem_u32(&full[i]), 1);
        fence_barrier_init();
    }
    __syncthreads();
    if (warp == 0)
        for (int k = 0; k < NN_STAGES; ++k) nn_issue(s, k, ring, full);
    int kbase = 0;
    for (int t = blockIdx.x; t < s.ntiles; t += gridDim.x, kbase += s.per_tile) {
        const long long r0 = (long long)t * NN_ROWS;
        const int nr = static_cast<int>(min((long long)NN_ROWS, s.r - r0));
        const double* zt = s.z + r0;
        double w[NN_CLASSES];
        // pass A: A1 in place in the ring, Z2 = A1 W2
        double z[NN_CLASSES];
#pragma unroll
        for (int j = 0; j < NN_CLASSES; ++j) z[j] = 0.0;
        for (int c = 0; c < s.nch; ++c) {
            const int k = kbase + c;
            nn_wait(full, k);
            const int c0 = c * NN_CHUNK, cw = min(NN_CHUNK, H - c0);
            double* st = ring + (k % NN_STAGES) * NN_STAGE_DOUBLES;
            if (lane < nr) {
                for (int hh = warp; hh < cw; hh += NN_WARPS) {
                    const int h = c0 + hh;
                    double* p = st + hh * NN_SLOT + piece_lead(zt + h * s.ld) + lane;
                    const double a = nn_sigmoid(*p);
                    if (resident) *p = a;
                    nn_w2_row(w, w2s, w2, ldw2, h, resident);
#pragma unroll
                    for (int j = 0; j < NN_CLASSES; ++j) z[j] = fma(a, w[j], z[j]);
                }
            }
            if (!resident) {
                __syncthreads();             // every warp has read the piece: the stage is free again
                if (warp == 0) nn_issue(s, k + NN_STAGES, ring, full);
            }
        }
#pragma unroll
        for (int j = 0; j < NN_CLASSES; ++j) zs[(warp * NN_ROWS + lane) * NN_CLASSES + j] = z[j];
        __syncthreads();
        // A2 = sigmoid(Z2), E2 = A2 - onehot(label), D2 = (1 - A2) A2 E2
        for (int i = tid; i < nr * NN_CLASSES; i += NN_THREADS) {
            double sum = zs[i];
            for (int q = 1; q < NN_WARPS; ++q) sum += zs[q * NN_ROWS * NN_CLASSES + i];
            const double a2 = nn_sigmoid(sum);
            const double e2 = labels[r0 + i / NN_CLASSES] == i % NN_CLASSES ? a2 - 1.0 : a2;
            d2s[i] = (1.0 - a2) * a2 * e2;
        }
        __syncthreads();
        // pass B: D1 = (1 - A1) A1 (D2 W2^T), then the partial of A1^T D2
        double d[NN_CLASSES];
#pragma unroll
        for (int j = 0; j < NN_CLASSES; ++j) d[j] = lane < nr ? d2s[lane * NN_CLASSES + j] : 0.0;
        for (int c = 0; c < s.nch; ++c) {
            const int k = kbase + (resident ? 0 : s.nch) + c;
            nn_wait(full, k);                // already complete for a resident tile
            const int c0 = c * NN_CHUNK, cw = min(NN_CHUNK, H - c0);
            double* st = ring + (k % NN_STAGES) * NN_STAGE_DOUBLES;
            if (lane < nr) {
                for (int hh = warp; hh < cw; hh += NN_WARPS) {
                    const int h = c0 + hh;
                    double* p = st + hh * NN_SLOT + piece_lead(zt + h * s.ld) + lane;
                    double a = *p;
                    if (!resident) *p = a = nn_sigmoid(a);
                    nn_w2_row(w, w2s, w2, ldw2, h, resident);
                    double e1 = 0.0;
#pragma unroll
                    for (int j = 0; j < NN_CLASSES; ++j) e1 = fma(d[j], w[j], e1);
                    d1[r0 + lane + h * ldd] = (1.0 - a) * a * e1;
                }
            }
            __syncthreads();
            // column hh of the piece, classes j0 .. j0 + nj - 1: acc += A1(r, h) * D2(r, j) over the rows in ascending order
            const int hh = tid >> 2, j0 = (tid & 3) * 3, nj = j0 < 9 ? 3 : 1;
            if (hh < cw) {
                const int h = c0 + hh;
                const double* col = st + hh * NN_SLOT + piece_lead(zt + h * s.ld);
                double acc[3];
#pragma unroll
                for (int i = 0; i < 3; ++i) acc[i] = i < nj ? mypart[h + (j0 + i) * H] : 0.0;
                for (int r = 0; r < nr; ++r) {
                    const double a = col[r];
#pragma unroll
                    for (int i = 0; i < 3; ++i)
                        if (i < nj) acc[i] = fma(a, d2s[r * NN_CLASSES + j0 + i], acc[i]);
                }
#pragma unroll
                for (int i = 0; i < 3; ++i)
                    if (i < nj) mypart[h + (j0 + i) * H] = acc[i];
            }
            __syncthreads();                 // the stage and (after the last piece) zs and d2s are free again
            if (warp == 0) {
                fence_proxy_async();
                nn_issue(s, k + NN_STAGES, ring, full);
            }
        }
    }
}

__global__ void __launch_bounds__(256)
nn_apply_kernel(const double* __restrict__ part, long long ldp, long long stride, const int* __restrict__ first, int nblocks,
                int rows, long long count, double scale, double* out, long long ldo, double* w, long long ldw) {
    const long long e = blockIdx.x * 256LL + threadIdx.x;
    if (e >= count) return;
    const long long i = e % rows, j = e / rows;
    const double* p = part + i + j * ldp;
    double total = 0.0;
    for (int b = 0; b < nblocks; ++b) {
        const int lo = first[b], hi = first[b + 1];
        double sum = p[lo * stride];
        for (int q = lo + 1; q < hi; ++q) sum = __dadd_rn(sum, p[q * stride]);
        const double scaled = __dmul_rn(sum, scale);
        total = b == 0 ? scaled : __dadd_rn(total, scaled);
    }
    if (out)
        out[i + j * ldo] = total;
    else
        w[i + j * ldw] = __dsub_rn(w[i + j * ldw], total);
}

}  // namespace

int nn_parts(int r, int num_sms) {
    const long long tiles = ((long long)r + NN_ROWS - 1) / NN_ROWS;
    return (int)(tiles < 1 ? 1 : (tiles < num_sms ? tiles : num_sms));
}

cudaError_t nn_backprop_f64(const double* z1, long long ld, int r, int H, const double* w2, long long ldw2, const int* labels,
                            double* d1, long long ldd, double* part, int num_sms, cudaStream_t st) {
    if (r <= 0 || H <= 0) return cudaErrorInvalidValue;
    NnShape s;
    s.z = z1;
    s.ld = ld;
    s.r = r;
    s.H = H;
    s.nch = (H + NN_CHUNK - 1) / NN_CHUNK;
    s.per_tile = H <= NN_RESIDENT_H ? s.nch : 2 * s.nch;
    s.ntiles = (int)(((long long)r + NN_ROWS - 1) / NN_ROWS);
    return launch_with_smem<nn_backprop_kernel>(nn_parts(r, num_sms), NN_THREADS, NN_SMEM, st, s, w2, ldw2, labels, d1, ldd, part);
}

cudaError_t nn_apply_f64(const double* part, long long ldp, long long stride, const int* first, int nblocks, int rows, int cols,
                         double scale, double* out, long long ldo, double* w, long long ldw, cudaStream_t st) {
    if (nblocks <= 0 || rows <= 0 || cols <= 0) return cudaErrorInvalidValue;
    const long long count = (long long)rows * cols;
    nn_apply_kernel<<<(unsigned)((count + 255) / 256), 256, 0, st>>>(part, ldp, stride, first, nblocks, rows, count, scale, out,
                                                                    ldo, w, ldw);
    return launched();
}

}  // namespace mb

// One ALS half-step (ml/ALSHelp.scala:292-382, updateBlock): for every entity u of the side being solved,
//   A_u = sum over u's ratings of y y^T  (+ numRatings * lambda on the diagonal, + YtY when implicit),  b_u = sum r y,
// then x_u = A_u^-1 b_u, where y runs over the fixed side's factor rows of u's rated partners.
//
// als_kernel<G, EPT, SOLVE>: a group of G threads works on one entity (G = 32, a warp, for rank <= 32; G = 256, the whole
// CTA, above).  Thread t of the group owns the packed-triangle elements e = t, t + G, ... (at most EPT of them, in
// registers; EPT is set per rank bucket: 2, 5 or 17 for a warp, 5 or 33 for a CTA) and b element t.  The entity's partner rows are gathered in chunks (max(16, 1024 / rank) rows) into the
// group's shared memory; each owned element then takes the chunk's terms in order, so every element is one sequential sum from 0.0 in the
// reference's order (product blocks ascending, product id ascending, then the ratings' input order, as the host lays out
// the links) with separate roundings: __dmul_rn / __dadd_rn, which are never contracted into DFMA, as the JVM never fuses.
//   explicit  A += fl(y_i y_j)                  (dspr onto zeros, then userXtX += tempXtX)
//             b += fl(r y_i)                    (axpy(r, y, Xy))
//   implicit  c = fl(1 + fl(alpha |r|)),  A += fl(fl(c - 1) fl(y_i y_j)),  b += fl(c y_i) only when r > 0
// Then A_ii += fl(n_u lambda) and, when implicit, A_ij += YtY_ij.  SOLVE = false writes A (packed lower, row-major) and b
// and stops: the bit-exact seam.  SOLVE = true factors A = L L^T in shared memory (right-looking, one column per step) and
// runs the two triangular solves there; A never reaches HBM.  A non-positive pivot (possible only with lambda = 0) marks
// the entity: its row is left unwritten and the lowest such entity id is kept in *bad.
// The host orders the work list heaviest first, so a long-tailed user starts early instead of ending the launch alone.
#include "als.h"
#include "launch.h"

#include <climits>

namespace mb {

constexpr int ALS_THREADS = 256;
constexpr int ALS_CHUNK_DOUBLES = 1024;  // a gathered chunk holds max(16, 1024 / rank) partner rows: fewer barriers per
                                         // term for small ranks, where one heavy entity would otherwise set the launch time
constexpr int ALS_MIN_CHUNK = 16;
constexpr int ALS_WARP_MAX_RANK = 32;    // one warp per entity up to this rank, one CTA per entity above
constexpr int ALS_MAX_RANK = 128;

struct AlsArgs {
    AlsLinks L;
    int rank;
    const double* Y;
    long long ldy;
    double lambda, alpha;
    int implicit;
    const double* yty;
    long long ldyty;
    double* X;          // SOLVE: the solved rows
    long long ldx;
    int* bad;
    double* A;          // !SOLVE: the packed triangles and right-hand sides
    double* B;
    int chunk;          // partner rows per gathered chunk
    int group_doubles;  // shared memory per group
};

__host__ __device__ constexpr int tri(int r) { return r * (r + 1) / 2; }

template <int G>
__device__ __forceinline__ void group_sync() {
    if constexpr (G == 32) __syncwarp();
    else __syncthreads();
}

// Outside an anonymous namespace, so the kernels' symbols (and profiler names) are stable.
template <int G, int EPT, bool SOLVE>
__global__ void __launch_bounds__(ALS_THREADS, 1) als_kernel(AlsArgs a) {
    extern __shared__ double smem[];
    constexpr int GROUPS = ALS_THREADS / G;
    const int grp = threadIdx.x / G, t = threadIdx.x % G;
    const long long k = (long long)blockIdx.x * GROUPS + grp;
    if (k >= a.L.count) return;                           // the whole group leaves together
    const int r = a.rank, T = tri(r);
    double* ys = smem + (size_t)grp * a.group_doubles;
    double* rs = ys + a.group_doubles - 2 * a.chunk;      // the chunk's ratings, after the rows (and the solve's space)
    int* ps = reinterpret_cast<int*>(rs + a.chunk);       // the chunk's partner rows
    const int pos = a.L.work[k];
    const long long p0 = a.L.offsets[pos], p1 = a.L.offsets[pos + 1];

    int ij[EPT];                                          // owned element e = t + q G is (i, j) = (ij >> 8, ij & 255)
    double acc[EPT];
#pragma unroll
    for (int q = 0; q < EPT; ++q) {
        const int e = t + q * G;
        int i = (int)((sqrtf(8.0f * (float)e + 1.0f) - 1.0f) * 0.5f);
        while (tri(i + 1) <= e) ++i;
        while (tri(i) > e) --i;
        ij[q] = (i << 8) | (e - tri(i));
        acc[q] = 0.0;
    }
    double bacc = 0.0;

    for (long long c0 = p0; c0 < p1; c0 += a.chunk) {
        const int rows = (int)min((long long)a.chunk, p1 - c0);
        group_sync<G>();                                  // the previous chunk has been consumed
        // two phases, so the row loads of the second do not wait on index loads one by one
        for (int q = t; q < rows; q += G) {
            ps[q] = a.L.partners[c0 + q];
            rs[q] = (double)a.L.ratings[c0 + q];          // exact widening
        }
        group_sync<G>();
#pragma unroll 4
        for (int x = t; x < rows * r; x += G) {
            const int row = x / r;
            ys[x] = a.Y[(long long)ps[row] * a.ldy + (x - row * r)];
        }
        group_sync<G>();
        for (int q = 0; q < rows; ++q) {
            const double* y = ys + q * r;
            const double rating = rs[q];
            if (!a.implicit) {
#pragma unroll
                for (int s = 0; s < EPT; ++s)
                    if (t + s * G < T) acc[s] = __dadd_rn(acc[s], __dmul_rn(y[ij[s] >> 8], y[ij[s] & 255]));
                if (t < r) bacc = __dadd_rn(bacc, __dmul_rn(rating, y[t]));
            } else {
                const double c = __dadd_rn(1.0, __dmul_rn(a.alpha, fabs(rating)));
                const double w = __dadd_rn(c, -1.0);
#pragma unroll
                for (int s = 0; s < EPT; ++s)
                    if (t + s * G < T) acc[s] = __dadd_rn(acc[s], __dmul_rn(w, __dmul_rn(y[ij[s] >> 8], y[ij[s] & 255])));
                if (t < r && rating > 0.0) bacc = __dadd_rn(bacc, __dmul_rn(c, y[t]));
            }
        }
    }

    // regularisation: numRatings * lambda (one Int x Double rounding) on the diagonal, then YtY when implicit
    const double reg = __dmul_rn((double)(p1 - p0), a.lambda);
#pragma unroll
    for (int s = 0; s < EPT; ++s) {
        const int i = ij[s] >> 8, j = ij[s] & 255;
        if (i == j) acc[s] = __dadd_rn(acc[s], reg);
        if (a.implicit && t + s * G < T) acc[s] = __dadd_rn(acc[s], a.yty[(long long)i * a.ldyty + j]);
    }

    if constexpr (!SOLVE) {
        double* A = a.A + (long long)pos * T;
#pragma unroll
        for (int s = 0; s < EPT; ++s)
            if (t + s * G < T) A[t + s * G] = acc[s];
        if (t < r) a.B[(long long)pos * r + t] = bacc;
        return;
    } else {
        double* Ls = ys;                                  // packed lower triangle, row-major
        double* bs = ys + T;
        double* zs = bs + r;
        group_sync<G>();                                  // every thread is done with the last chunk
#pragma unroll
        for (int s = 0; s < EPT; ++s)
            if (t + s * G < T) Ls[t + s * G] = acc[s];
        if (t < r) bs[t] = bacc;
        // Cholesky, one column per step: scale column k by sqrt(L_kk), then update the trailing triangle
        for (int kk = 0; kk < r; ++kk) {
            group_sync<G>();
            const double d = Ls[tri(kk) + kk];
            if (!(d > 0.0)) {                             // every thread of the group read the same pivot
                if (t == 0) atomicMin(a.bad, a.L.ids[pos]);
                return;
            }
            const double sd = sqrt(d);
#pragma unroll
            for (int s = 0; s < EPT; ++s) {
                const int i = ij[s] >> 8, j = ij[s] & 255;
                if (t + s * G < T && j == kk && i > kk) Ls[t + s * G] = Ls[t + s * G] / sd;
            }
            group_sync<G>();
#pragma unroll
            for (int s = 0; s < EPT; ++s) {
                const int i = ij[s] >> 8, j = ij[s] & 255;
                if (t + s * G < T && j > kk) Ls[t + s * G] -= Ls[tri(i) + kk] * Ls[tri(j) + kk];
            }
            if (t == 0) Ls[tri(kk) + kk] = sd;           // read again only after the next step's barrier
        }
        // L z = b (z in zs), then L^T x = z (x in bs); one barrier per step, each step writes only entries it does not read
        for (int kk = 0; kk < r; ++kk) {
            group_sync<G>();
            const double z = bs[kk] / Ls[tri(kk) + kk];
            if (t == 0) zs[kk] = z;
            for (int i = kk + 1 + t; i < r; i += G) bs[i] -= Ls[tri(i) + kk] * z;
        }
        for (int kk = r - 1; kk >= 0; --kk) {
            group_sync<G>();
            const double x = zs[kk] / Ls[tri(kk) + kk];
            if (t == 0) bs[kk] = x;
            for (int i = t; i < kk; i += G) zs[i] -= Ls[tri(kk) + i] * x;
        }
        group_sync<G>();
        if (t < r) a.X[(long long)pos * a.ldx + t] = bs[t];
    }
}

__global__ void coo_scatter_kernel(long long nnz, const int32_t* row, const int32_t* col, const float* val, double* out,
                                   long long ld) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e < nnz) out[(long long)row[e] * ld + col[e]] = (double)val[e];
}

namespace {

template <int G, int EPT, bool SOLVE>
cudaError_t launch(AlsArgs a, cudaStream_t st) {
    constexpr int GROUPS = ALS_THREADS / G;
    const int r = a.rank;
    a.chunk = ALS_CHUNK_DOUBLES / r > ALS_MIN_CHUNK ? ALS_CHUNK_DOUBLES / r : ALS_MIN_CHUNK;
    a.group_doubles = (SOLVE ? (tri(r) > a.chunk * r ? tri(r) : a.chunk * r) + 2 * r : a.chunk * r) + 2 * a.chunk;
    const size_t smem = (size_t)GROUPS * a.group_doubles * sizeof(double);
    cudaError_t e = cudaFuncSetAttribute(als_kernel<G, EPT, SOLVE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const long long grid = (a.L.count + GROUPS - 1) / GROUPS;
    als_kernel<G, EPT, SOLVE><<<(unsigned)grid, ALS_THREADS, smem, st>>>(a);
    return launched();
}

template <bool SOLVE>
cudaError_t dispatch(const AlsArgs& a, cudaStream_t st) {
    if (a.L.count <= 0) return cudaSuccess;
    if (a.rank < 1 || a.rank > ALS_MAX_RANK) return cudaErrorInvalidValue;
    // EPT (owned triangle elements per thread) sized to the rank's bucket, so few unrolled slots sit predicated off
    if (a.rank <= 10) return launch<32, (tri(10) + 31) / 32, SOLVE>(a, st);
    if (a.rank <= 17) return launch<32, (tri(17) + 31) / 32, SOLVE>(a, st);
    if (a.rank <= ALS_WARP_MAX_RANK) return launch<32, (tri(ALS_WARP_MAX_RANK) + 31) / 32, SOLVE>(a, st);
    if (a.rank <= 50) return launch<ALS_THREADS, (tri(50) + ALS_THREADS - 1) / ALS_THREADS, SOLVE>(a, st);
    return launch<ALS_THREADS, (tri(ALS_MAX_RANK) + ALS_THREADS - 1) / ALS_THREADS, SOLVE>(a, st);
}

}  // namespace

cudaError_t als_solve(const AlsLinks& L, int rank, const double* Y, long long ldy, double lambda, double alpha, bool implicit,
                      const double* yty, long long ldyty, double* X, long long ldx, int* bad, cudaStream_t st) {
    AlsArgs a{L, rank, Y, ldy, lambda, alpha, implicit ? 1 : 0, yty, ldyty, X, ldx, bad, nullptr, nullptr, 0, 0};
    return dispatch<true>(a, st);
}

cudaError_t als_assemble(const AlsLinks& L, int rank, const double* Y, long long ldy, double lambda, double alpha,
                         bool implicit, const double* yty, long long ldyty, double* A, double* B, cudaStream_t st) {
    AlsArgs a{L, rank, Y, ldy, lambda, alpha, implicit ? 1 : 0, yty, ldyty, nullptr, 0, nullptr, A, B, 0, 0};
    return dispatch<false>(a, st);
}

cudaError_t coo_scatter_rows(long long nnz, const int32_t* row, const int32_t* col, const float* val, double* out,
                             long long ld, cudaStream_t st) {
    if (nnz <= 0) return cudaSuccess;
    coo_scatter_kernel<<<(unsigned)((nnz + 255) / 256), 256, 0, st>>>(nnz, row, col, val, out, ld);
    return launched();
}

}  // namespace mb

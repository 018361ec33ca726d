// Symmetric eigensolver — the eigen step of DenseVecMatrix.computeSVD (matrix/DenseVecMatrix.scala:1589-1606), which the
// reference hands to LAPACK (brzSvd = dgesdd of the Gramian) or ARPACK (symmetricEigs, :1725-1834).
//
// Parallel cyclic two-sided Jacobi on a working copy of G (n padded to even N with a zero row / column):
//   * round-robin ordering: position 2a and 2a+1 form pair a.  A round rotates all N/2 pairs at once; between rounds the
//     positions move by the circle method (position 0 fixed, the others on one cycle of length N-1), so a sweep of N-1
//     rounds meets every index pair once and ends with every index back at its own position;
//   * one kernel per round (jacobi_round_kernel): every CTA computes the rotations (Rutishauser's stable formulas, skipped
//     when |g_pq| <= eps * sqrt(|g_pp g_qq|)) of the pairs it touches from the round's input, then updates its 2x2 blocks
//     G_ab <- R_a^T G_ab R_b and the column pairs V_b <- V_b R_b, storing them to their next-round positions in the other
//     buffer of a ping-pong pair;
//   * every element of G_ab is a four-term sum taken in an order that is the same for G_ba, with rounding fixed
//     (__dmul_rn / __dadd_rn, never contracted), so the working matrix stays exactly symmetric;
//   * a sweep (memset of the "rotated" flag, N-1 rounds, copy of the flag to the host) is one CUDA graph; the host stops
//     after the first sweep that rotated nothing.
// No atomics, no reductions across threads: the result is bitwise reproducible from run to run.
#include "eigen.h"

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <numeric>
#include <vector>

namespace mb {

namespace {

constexpr int TP = 16;        // pairs per CTA side: a CTA updates a 16 x 16 grid of 2x2 blocks (32 x 32 elements)

__device__ __forceinline__ int next_pos(int p, int m) {
    if (m < 2) return p;
    const int a = p >> 1;
    if ((p & 1) == 0) {                        // top[a]: top[0] stays, top[a] -> top[a+1], top[m-1] -> bot[m-1]
        if (a == 0) return 0;
        return a == m - 1 ? 2 * a + 1 : 2 * (a + 1);
    }
    return a == 0 ? 2 : 2 * (a - 1) + 1;       // bot[0] -> top[1], bot[a] -> bot[a-1]
}

__global__ void __launch_bounds__(256) jacobi_init_kernel(const double* __restrict__ G, long long rs, long long cs, int n, int N,
                                                          double* __restrict__ W, double* __restrict__ V) {
    const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (e >= (long long)N * N) return;
    const int i = (int)(e % N), j = (int)(e / N);
    double g = 0.0;
    if (i < n && j < n) g = i >= j ? G[i * rs + j * cs] : G[j * rs + i * cs];     // lower triangle, mirrored
    W[e] = g;
    V[e] = i == j ? 1.0 : 0.0;
}

// grid.x: (m/16 rounded up)^2 tiles, grid.y: 0 = G, 1 = V.  Both matrices are N x N, column-major, ld = N.
__global__ void __launch_bounds__(256) jacobi_round_kernel(const double* __restrict__ Gin, double* __restrict__ Gout,
                                                           const double* __restrict__ Vin, double* __restrict__ Vout, int N,
                                                           int* __restrict__ rotated) {
    __shared__ double s_c[2 * TP], s_s[2 * TP], s_t[2 * TP];
    __shared__ int s_rot[2 * TP];
    const int m = N >> 1;
    const int tiles = (m + TP - 1) / TP;
    const int a0 = (blockIdx.x % tiles) * TP, b0 = (blockIdx.x / tiles) * TP;
    const bool is_v = blockIdx.y == 1;
    const long long ld = N;
    if (threadIdx.x < 2 * TP) {
        // rotation of pair `a` (row side for threads 0..15, column side for 16..31): one call site, so every CTA that needs
        // the rotation of a pair computes it with the same instructions from the same inputs
        const int a = threadIdx.x < TP ? a0 + threadIdx.x : b0 + threadIdx.x - TP;
        double c = 1.0, s = 0.0, t = 0.0;
        int rot = 0;
        if (a < m) {
            const double gpp = Gin[2 * a + 2 * a * ld], gqq = Gin[2 * a + 1 + (2 * a + 1) * ld];
            const double gpq = Gin[2 * a + 1 + 2 * a * ld];
            if (!(fabs(gpq) <= DBL_EPSILON * sqrt(fabs(gpp * gqq)))) {
                const double th = (gqq - gpp) / (2.0 * gpq);
                t = fabs(th) > 1e150 ? 0.5 / th : (th >= 0.0 ? 1.0 : -1.0) / (fabs(th) + sqrt(1.0 + th * th));
                c = 1.0 / sqrt(1.0 + t * t);
                s = t * c;
                rot = 1;
            }
        }
        s_c[threadIdx.x] = c;
        s_s[threadIdx.x] = s;
        s_t[threadIdx.x] = t;
        s_rot[threadIdx.x] = rot;
        if (rot && !is_v && threadIdx.x < TP && blockIdx.x < tiles) *rotated = 1;
    }
    __syncthreads();
    const int ta = threadIdx.x & (TP - 1), tb = threadIdx.x >> 4;
    const int a = a0 + ta, b = b0 + tb;
    if (a >= m || b >= m) return;
    const double cb = s_c[TP + tb], sb = s_s[TP + tb];
    const int p0 = next_pos(2 * a, m), p1 = next_pos(2 * a + 1, m);
    const int q0 = next_pos(2 * b, m), q1 = next_pos(2 * b + 1, m);
    if (is_v) {
        // V_b <- V_b R_b on rows 2a, 2a+1; rows keep their place, columns move
        const double2 x0 = *reinterpret_cast<const double2*>(Vin + 2 * a + 2 * b * ld);          // column 2b
        const double2 x1 = *reinterpret_cast<const double2*>(Vin + 2 * a + (2 * b + 1) * ld);    // column 2b+1
        *reinterpret_cast<double2*>(Vout + 2 * a + q0 * ld) = make_double2(cb * x0.x - sb * x1.x, cb * x0.y - sb * x1.y);
        *reinterpret_cast<double2*>(Vout + 2 * a + q1 * ld) = make_double2(sb * x0.x + cb * x1.x, sb * x0.y + cb * x1.y);
        return;
    }
    const double2 x0 = *reinterpret_cast<const double2*>(Gin + 2 * a + 2 * b * ld);
    const double2 x1 = *reinterpret_cast<const double2*>(Gin + 2 * a + (2 * b + 1) * ld);
    double z[2][2];
    if (a == b) {
        // the rotated pair itself: Rutishauser's update of the diagonal, the off-diagonal entry annihilated
        if (s_rot[ta]) {
            const double t = s_t[ta], gpq = x0.y;
            z[0][0] = x0.x - t * gpq;
            z[1][1] = x1.y + t * gpq;
            z[0][1] = z[1][0] = 0.0;
        } else {
            z[0][0] = x0.x; z[1][0] = x0.y; z[0][1] = x1.x; z[1][1] = x1.y;
        }
    } else {
        const double ca = s_c[ta], sa = s_s[ta];
        const double Ra[2][2] = {{ca, sa}, {-sa, ca}}, Rb[2][2] = {{cb, sb}, {-sb, cb}};
        const double X[2][2] = {{x0.x, x1.x}, {x0.y, x1.y}};
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                // z_ij = sum_kl Ra[k][i] Rb[l][j] X[k][l], summed as (kl=00 + kl=11) + (kl=01 + kl=10): the same value as
                // element (j, i) of block (b, a), computed by another thread
                const double t00 = __dmul_rn(__dmul_rn(Ra[0][i], Rb[0][j]), X[0][0]);
                const double t11 = __dmul_rn(__dmul_rn(Ra[1][i], Rb[1][j]), X[1][1]);
                const double t01 = __dmul_rn(__dmul_rn(Ra[0][i], Rb[1][j]), X[0][1]);
                const double t10 = __dmul_rn(__dmul_rn(Ra[1][i], Rb[0][j]), X[1][0]);
                z[i][j] = __dadd_rn(__dadd_rn(t00, t11), __dadd_rn(t01, t10));
            }
    }
    Gout[p0 + q0 * ld] = z[0][0];
    Gout[p1 + q0 * ld] = z[1][0];
    Gout[p0 + q1 * ld] = z[0][1];
    Gout[p1 + q1 * ld] = z[1][1];
}

// out(i, j) = V[i + order[j] * ld] for i, j < n
__global__ void __launch_bounds__(256) jacobi_gather_kernel(const double* __restrict__ V, long long ld, const int* __restrict__ order,
                                                            int n, double* __restrict__ out, long long rs, long long cs) {
    const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (e >= (long long)n * n) return;
    const int i = (int)(e % n), j = (int)(e / n);
    out[i * rs + j * cs] = V[i + order[j] * ld];
}

struct Buffers {
    double* W[2] = {nullptr, nullptr};
    double* V[2] = {nullptr, nullptr};
    int* flag = nullptr;
    int* flag_host = nullptr;
    int* order = nullptr;
    cudaGraphExec_t exec[2] = {nullptr, nullptr};
    ~Buffers() {
        for (int i = 0; i < 2; ++i) {
            if (W[i]) cudaFree(W[i]);
            if (V[i]) cudaFree(V[i]);
            if (exec[i]) cudaGraphExecDestroy(exec[i]);
        }
        if (flag) cudaFree(flag);
        if (flag_host) cudaFreeHost(flag_host);
        if (order) cudaFree(order);
    }
};

// one sweep starting from buffer `from`: clear the flag, N-1 rounds, flag -> host
cudaError_t capture_sweep(Buffers& B, int N, int from, cudaGraphExec_t* exec) {
    cudaStream_t cs = nullptr;
    cudaError_t e = cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking);
    if (e != cudaSuccess) return e;
    cudaGraph_t graph = nullptr;
    e = cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal);
    if (e == cudaSuccess) {
        cudaMemsetAsync(B.flag, 0, sizeof(int), cs);
        const int m = N / 2, tiles = (m + TP - 1) / TP;
        int cur = from;
        for (int r = 0; r < N - 1; ++r) {
            jacobi_round_kernel<<<dim3(tiles * tiles, 2), 256, 0, cs>>>(B.W[cur], B.W[cur ^ 1], B.V[cur], B.V[cur ^ 1], N, B.flag);
            cur ^= 1;
        }
        cudaMemcpyAsync(B.flag_host, B.flag, sizeof(int), cudaMemcpyDeviceToHost, cs);
        const cudaError_t e2 = cudaStreamEndCapture(cs, &graph);
        e = e2 != cudaSuccess ? e2 : cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaGraphInstantiate(exec, graph, 0);
    if (graph) cudaGraphDestroy(graph);
    cudaStreamDestroy(cs);
    return e;
}

}  // namespace

cudaError_t syev_jacobi(int n, const double* G, long long rs, long long cs, double* V, long long vrs, long long vcs,
                        double* w_host, int* sweeps, int max_sweeps, cudaStream_t stream, long long* launches) {
    if (sweeps) *sweeps = 0;
    if (n <= 0) return cudaSuccess;
    const int N = n + (n & 1);
    const size_t bytes = (size_t)N * N * sizeof(double);
    Buffers B;
    cudaError_t e;
    for (int i = 0; i < 2; ++i) {
        if ((e = cudaMalloc(&B.W[i], bytes)) != cudaSuccess) return e;
        if ((e = cudaMalloc(&B.V[i], bytes)) != cudaSuccess) return e;
    }
    if ((e = cudaMalloc(&B.flag, sizeof(int))) != cudaSuccess) return e;
    if ((e = cudaMallocHost(&B.flag_host, sizeof(int))) != cudaSuccess) return e;
    if ((e = cudaMalloc(&B.order, sizeof(int) * n)) != cudaSuccess) return e;
    const long long total = (long long)N * N;
    jacobi_init_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(G, rs, cs, n, N, B.W[0], B.V[0]);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    if (launches) ++*launches;
    int cur = 0, done = 0;
    for (int sw = 1; sw <= max_sweeps; ++sw) {
        if (!B.exec[cur] && (e = capture_sweep(B, N, cur, &B.exec[cur])) != cudaSuccess) return e;
        if ((e = cudaGraphLaunch(B.exec[cur], stream)) != cudaSuccess) return e;
        if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return e;
        if (launches) *launches += N - 1;
        cur ^= (N - 1) & 1;
        if (sweeps) *sweeps = sw;
        if (*B.flag_host == 0) { done = 1; break; }
    }
    if (!done) return cudaErrorNotReady;
    // after whole sweeps every index is back at its own position: the eigenvalues are the diagonal of W[cur]
    std::vector<double> w(n);
    if ((e = cudaMemcpy2DAsync(w.data(), sizeof(double), B.W[cur], (N + 1) * sizeof(double), sizeof(double), n,
                               cudaMemcpyDeviceToHost, stream)) != cudaSuccess)
        return e;
    if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return e;
    std::vector<int> order(n);
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return std::fabs(w[x]) > std::fabs(w[y]); });
    for (int j = 0; j < n; ++j) w_host[j] = w[order[j]];
    if ((e = cudaMemcpyAsync(B.order, order.data(), sizeof(int) * n, cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
    const long long nn = (long long)n * n;
    jacobi_gather_kernel<<<(unsigned)((nn + 255) / 256), 256, 0, stream>>>(B.V[cur], N, B.order, n, V, vrs, vcs);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    if (launches) ++*launches;
    return cudaStreamSynchronize(stream);     // the buffers are freed on return
}

}  // namespace mb

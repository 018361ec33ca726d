#pragma once
#include <cuda_runtime.h>

namespace mb {

// C (M x N, col-major, ldc) = alpha * op(A) * op(B) + beta * C, fp64.
// op(X) = X or X^T; A is stored (M x K) if !transA else (K x M); B likewise (K x N) / (N x K).
// Dispatches the TMA + DMMA tensor-core kernel when pointers are 16B aligned and leading
// dimensions are even, otherwise (or if force_generic) the CUDA-core kernel.
cudaError_t gemm_f64(bool transA, bool transB, int M, int N, int K, double alpha, const double* A, long long lda,
                     const double* B, long long ldb, double beta, double* C, long long ldc, int num_sms,
                     cudaStream_t stream, bool force_generic);

// One persistent launch for a blocked multiply: C[c] = sum_kk A[i*k+kk] * B[kk*n+j] for every c = i*n+j in my_c
// (all 'N' column-major blocks).  Returns cudaErrorNotSupported when the group does not fit the fixed-size parameter
// block or an operand is not TMA-addressable; the caller then falls back to one launch per block product.
cudaError_t gemm_f64_grouped(int m, int k, int n, const int* my_c, int num_c, const double* const* A, const long long* lda,
                             const double* const* B, const long long* ldb, double* const* C, const long long* ldc,
                             const int* row_len, const int* k_len, const int* col_len, int num_sms, cudaStream_t stream);

// ---- the general grouped launch (see gemm_f64.cu): entries = regions of C blocks with their own K segment lists,
//      operand readiness flags, optional staged addend (D = acc + Cin) and completion signals ----
constexpr int G2_MAX_OPS = 32;        // operand tiles per side
constexpr int G2_MAX_ENTRIES = 64;
constexpr int G2_MAX_SEG = 16;        // K segments (kk) per entry

struct G2Operand {                    // one column-major operand tile: A(i,kk) is rows x cols = M_i x K_kk, B(kk,j) is K_kk x N_j
    const double* ptr = nullptr;
    long long ld = 0;
    int rows = 0, cols = 0;
    int band = 0;                     // A: rows per readiness band, B: columns per band (multiples of 128); 0 = resident
    int ready_base = -1;              // index of the tile's first band flag in G2Launch::ready, -1 = resident (never polled)
};
struct G2Entry {
    int nseg = 0;
    int a_op[G2_MAX_SEG] = {}, b_op[G2_MAX_SEG] = {};   // operand indices of K segment s
    int m_off = 0, n_off = 0, M = 0, N = 0;             // region inside the C block (offsets are multiples of 128)
    double* D = nullptr;                                // output, element (m_off, n_off) of the region; may be a peer pointer
    long long ldd = 0;
    const double* Cin = nullptr;                        // optional addend: D = acc + Cin
    long long ldcin = 0;
    bool sub_from_cin = false;                          // D = Cin - acc instead (Cin required, no cin_flag; D == Cin
                                                        // allowed); every entry of one launch must agree
    const unsigned long long* cin_flag = nullptr;       // wait until *cin_flag >= cin_val (system scope) before reading Cin
    unsigned long long cin_val = 0;
    unsigned long long* done_ctr = nullptr;             // zeroed device counter; when it reaches the entry's tile count ...
    unsigned long long* sig_local = nullptr;            // ... this flag is set to sig_val (st.release.sys); D must be local
    unsigned long long sig_val = 0;
};
struct G2Launch {
    int na = 0, nb = 0, ne = 0;
    G2Operand A[G2_MAX_OPS], B[G2_MAX_OPS];
    G2Entry E[G2_MAX_ENTRIES];
    const unsigned long long* ready = nullptr;          // band flags (device memory), "landed" means >= ready_val
    unsigned long long ready_val = 0;
    unsigned long long* status = nullptr;               // device word set to 1 when an in-kernel wait times out
    long long timeout_ns = 0;                           // 0 = wait forever
};
cudaError_t gemm_f64_grouped2(const G2Launch& L, int num_sms, cudaStream_t stream);

// Gramian: G (n x n, col-major, ldg) = op(A) op(A)^T with op(A) n x K (A stored n x K if !trans, K x n if trans), exactly
// symmetric.  TMA-addressable operands run the DMMA mainloop over the lower-triangle tiles only; when the triangle has
// too few tiles for the SMs, K is split into gram_splits() partials held in `ws`.  The rest run the CUDA-core GEMM.  One
// fixed-order pass then sums the partials and mirrors them (in place in G when there is one split).
// ws: gram_workspace_doubles(n, K, num_sms) doubles, 16-byte aligned; 0 (ws may be null) unless K is split, and never
// more than GRAM_WS_CAP_DOUBLES.
constexpr long long GRAM_WS_CAP_DOUBLES = 32LL << 20;    // 256 MiB
int gram_splits(int n, long long K, int num_sms);
size_t gram_workspace_doubles(int n, long long K, int num_sms);
cudaError_t gram_f64(bool trans, int n, int K, const double* A, long long lda, double* G, long long ldg, double* ws,
                     int num_sms, cudaStream_t stream);

bool gemm_f64_tma_eligible(const double* A, long long lda, const double* B, long long ldb);

}  // namespace mb

#pragma once
#include <cuda_runtime.h>

namespace mb {

// A CSC block on the device: column j holds rowidx/vals[colptr[j] .. colptr[j+1]), row indices strictly increasing.
struct CscView {
    int rows, cols;
    const int* colptr;
    const int* rowidx;
    const double* vals;
};
// A CSR copy of the same block (rows ascending, column indices strictly increasing within a row).
struct CsrView {
    int rows, cols;
    const int* rowptr;
    const int* colidx;
    const double* vals;
};
// A dense view: element (r, c) at p[r * rs + c * cs].
struct DView {
    double* p;
    long long rs, cs;
};

// out (rows x cols view) = S, zeros where nothing is stored.
cudaError_t csc_to_dense(const CscView& S, DView out, cudaStream_t st);
// C (m x n) [+]= A (m x K, dense) * B (K x n, CSC); each C(r, j) summed over B's column j in stored order.
cudaError_t spmm_dense_sparse(int m, DView A, const CscView& B, DView C, bool accumulate, cudaStream_t st);
// Builds the CSR copy of S into rowptr (rows + 1), colidx (nnz), vals (nnz); deterministic.
cudaError_t csc_to_csr(const CscView& S, long long nnz, int* rowptr, int* colidx, double* vals, cudaStream_t st);
// C (m x n) [+]= A (m x K, CSR copy) * B (K x n, dense); each C(r, j) summed over k ascending.
cudaError_t spmm_sparse_dense(const CsrView& A, int n, DView B, DView C, bool accumulate, cudaStream_t st);
// C (m x n, dense) [+]= A (m x K, CSC) * B (K x n, CSC); each C(r, j) summed over B's column j in stored order.
cudaError_t spgemm_dense_out(const CscView& A, const CscView& B, DView C, bool accumulate, cudaStream_t st);
// Row indices of the sparse generator: column j takes s rows by selection sampling from stream positions
// [first + j*rows, first + (j+1)*rows) of the XORShift stream state0; colptr[j] = j*s.
cudaError_t sparse_sample_rows(int rows, int cols, int s, unsigned long long state0, long long first, int* colptr,
                               int* rowidx, cudaStream_t st);

}  // namespace mb

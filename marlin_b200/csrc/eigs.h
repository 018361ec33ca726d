// y = A^T (A x) over a row-major fp64 view in one pass: the operator of computeSVD's dist-eigs mode
// (DenseVecMatrix.multiplyGramianMatrixBy, matrix/DenseVecMatrix.scala:1444-1459).
#pragma once
#include <cuda_runtime.h>

namespace mb {

// Partial vectors (of n doubles each) the product needs for m rows: the workspace is gram_matvec_parts(m) * n doubles.
int gram_matvec_parts(long long m, int n, int num_sms);
// a: row r at a + r * lda (8-byte aligned, any lda >= n); x[j * incx]; y[j * incy] = (accumulate ? y + : ) A^T (A x).
// m = 0 writes zeros (or leaves y when accumulating).  Two launches when m > 0.
cudaError_t gram_matvec_f64(const double* a, long long lda, long long m, int n, const double* x, long long incx, double* y,
                            long long incy, bool accumulate, double* part, int num_sms, cudaStream_t st);

}  // namespace mb

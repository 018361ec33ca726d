#pragma once
#include <cuda_runtime.h>
#include <cstddef>

namespace mb {

// y (len m, or n when trans) = A x [+ y]; A column-major m x n with leading dimension lda.  `workspace` holds
// gemv_workspace_doubles(trans, m, n) doubles of partial vectors.
size_t gemv_workspace_doubles(bool trans, int m, int n);
cudaError_t gemv_f64(bool trans, int m, int n, const double* a, long long lda, const double* x, long long incx, double* y,
                     long long incy, bool accumulate, double* workspace, cudaStream_t st);
// out (column-major m x n, ldo) = x y^T
cudaError_t ger_f64(int m, int n, const double* x, long long incx, const double* y, long long incy, double* out,
                    long long ldo, cudaStream_t st);
// scratch[0] = sum_i x_i y_i  (scratch holds dot_scratch_doubles() doubles)
int dot_scratch_doubles();
cudaError_t dot_f64(long long n, const double* x, long long incx, const double* y, long long incy, double* scratch,
                    cudaStream_t st);

}  // namespace mb

#pragma once
#include <cuda_runtime.h>

namespace mb {

// A strided fp64 view: element (r, c) at p[r*rs + c*cs] (column-major: rs = 1, cs = ld; transposed view: rs = ld, cs = 1).
struct FView {
    double* p;
    long long rs, cs;
    int rows, cols;
};

// LU with partial pivoting in place (LAPACK dgetrf conventions: unit-lower L and U packed, first maximal |a| pivots).
// piv_dev[i] (i < min(m, n)): 0-based row interchanged with row i; perm_dev (optional, n ints): row i of P*A is row
// perm[i] of A; info_dev: 0, or 1 + the first column whose pivot is exactly zero.
cudaError_t getrf(const FView& a, int* piv_dev, int* perm_dev, int* info_dev, int num_sms, cudaStream_t st);
// Cholesky A = L L^T in place: L in the lower triangle, strict upper triangle zeroed (Breeze `cholesky`); only the lower
// triangle of the input is read.  info_dev: 0, or 1 + the first row whose pivot is not positive.
cudaError_t potrf_lower(const FView& a, int* info_dev, int num_sms, cudaStream_t st);
// out = A^-1 from the packed LU factors of A and their interchanges.
cudaError_t inverse_from_lu(const FView& lu, const int* piv_dev, const FView& out, int num_sms, cudaStream_t st);
// T X = B in place (T triangular, left side); right-side solves are left-side solves of the transposed views.
cudaError_t trsm_left(const FView& T, bool lower, bool unit, const FView& B, int num_sms, cudaStream_t st);

}  // namespace mb

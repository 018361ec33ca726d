#pragma once
#include <cuda_runtime.h>

namespace mb {

// Symmetric eigendecomposition of the n x n view G (element (i, j) at G[i * rs + j * cs]; only the lower triangle is read)
// by parallel cyclic two-sided Jacobi.  On success w_host[0..n) holds the eigenvalues ordered by |w| descending (ties:
// lower index first) and V (n x n view, strides vrs / vcs) the matching orthonormal eigenvectors as columns.  *sweeps is the
// number of sweeps run, the last of which applied no rotation.  Returns cudaErrorNotReady when `max_sweeps` sweeps did not
// converge (w_host and V are then left unset).  Blocking: returns after the result is on the host / in V.
cudaError_t syev_jacobi(int n, const double* G, long long rs, long long cs, double* V, long long vrs, long long vcs,
                        double* w_host, int* sweeps, int max_sweeps, cudaStream_t stream, long long* launches);

}  // namespace mb

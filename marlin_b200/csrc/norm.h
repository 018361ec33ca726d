// DenseVecMatrix.norm (matrix/DenseVecMatrix.scala:975-999): one pass over an fp64 view for the 1-, infinity- and
// Frobenius norms.  See norm.cu.
#pragma once
#include <cuda_runtime.h>

namespace mb {

enum NormKind { NORM_ONE = 0, NORM_INF = 1, NORM_FRO = 2 };

// Bytes of device memory norm_f64 needs for an m x n view in `kind`: the chunk partials plus the results.
size_t norm_workspace_bytes(int kind, long long m, int n);

// Element (r, c) of the m x n view is x[r * rs + c * cs].  m > 0 and n > 0.  `ws` holds norm_workspace_bytes.
//   NORM_ONE: col[j * inc] = sum over rows of |x_rj| (chunks of NORM_CHUNK rows summed in row order, then the chunk
//             partials in chunk order); result[0] = the largest of them.
//   NORM_INF: result[0] = the largest row sum of |x| (each a left fold in column order from 0.0).
//   NORM_FRO: result[0..2] = Blue's small, medium and big accumulators of sum x^2 (see norm_fro_finish).
// The largest value follows java.lang.Double.compare: a NaN is larger than everything.  Every result is the same bits on
// every run.  `result` points into ws (device memory).
cudaError_t norm_f64(int kind, const double* x, long long rs, long long cs, long long m, int n, double* col, long long inc,
                     void* ws, double** result, int num_sms, cudaStream_t st);

}  // namespace mb

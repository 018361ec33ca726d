// DenseVecMatrix.lr (matrix/DenseVecMatrix.scala:1005-1035): the gradient of one logistic-regression step over a row-major
// fp64 shard, and the weight update.
#pragma once
#include <cuda_runtime.h>
#include <cstddef>

namespace mb {

// Number of per-CTA partial gradients lr_gradient_f64 writes for m rows (its grid size).
int lr_parts(int m, int num_sms);

// x: m x n row-major (row r at x + r * ld, any ld >= n, 8-byte aligned).  Column 0 is the label and counts as 1 in the
// features.  part: lr_parts(m, num_sms) * n doubles of workspace.  w, out: n doubles on the device.
//   update == false: out = sum over rows of x~_r * g_r,  g_r = 1 / (1 + exp(-(x~_r . w))) - x_r0
//   update == true:  w = w - (that sum) * scale  (out unused)
// The margins are sequential in column order with separate multiplies and adds; the sum is per CTA in ascending row
// order, then over CTAs in ascending order.  Two launches.
cudaError_t lr_gradient_f64(const double* x, long long ld, int m, int n, double* w, double* part, double* out, bool update,
                            double scale, int num_sms, cudaStream_t st);

}  // namespace mb

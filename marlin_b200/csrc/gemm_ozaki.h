#pragma once
#include <cuda_runtime.h>
#include <cstddef>

namespace mb {

// C (M x N, column-major fp64) = A * B (+ C), A (M x K) and B (K x N) column-major fp64, computed on the int8 tensor
// cores from `s` 7-bit digit planes per operand (see gemm_ozaki.cu).  `workspace` must hold ozaki_workspace_bytes().
size_t ozaki_workspace_bytes(int M, int N, int K, int s);
bool ozaki_supported(int M, int N, int K, int s, int bits);
cudaError_t gemm_f64_ozaki(int M, int N, int K, const double* A, long long lda, const double* B, long long ldb, double* C,
                           long long ldc, bool accumulate, int s, int bits, void* workspace, int num_sms, cudaStream_t stream);

}  // namespace mb

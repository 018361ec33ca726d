#pragma once
#include <cuda_runtime.h>

namespace mb {

// C (M x N col-major, ldc; fp32 or bf16) = sum_s op(A_s) * op(B_s) (+ C if accumulate), bf16 operands, fp32 accumulation
// in registers (wgmma.mma_async, f32 += bf16 x bf16); A_s stored (M x K_s) if !transA else (K_s x M).  The contraction
// is split into `nseg` (1..8) segments so the kk-sum of a blocked multiply is one launch per C block (the accumulator
// stays in registers; no read-modify-write of C).  The operands are read by TMA: every A_s / B_s must be 16-byte aligned
// with ld % 8 == 0 and every K_s > 0, else cudaErrorNotSupported (nothing launched).  C has no alignment rule.
// bf16_gemm in capi.cu stages operands that break the rule, handles K = 0 and caps fp32 accumulation chains.
cudaError_t gemm_bf16_segments(bool transA, bool transB, int M, int N, int nseg, const int* Kseg, const void* const* A,
                               const long long* lda, const void* const* B, const long long* ldb, void* C, long long ldc,
                               bool c_is_f32, bool accumulate, int num_sms, cudaStream_t stream);

}  // namespace mb

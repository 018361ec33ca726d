#pragma once
#include <cuda_runtime.h>

namespace mb {

enum { EW_ADD = 0, EW_SUB = 1, EW_MUL = 2 };               // binary ops
enum { EW_AXPB = 10, EW_DIV = 11, EW_RDIV = 12, EW_COPY = 13, EW_FILL = 14 };   // unary ops (EW_FILL: out = beta)

// A view's element (r,c) lives at base[r*rs + c*cs]  (col-major: rs=1, cs=ld; transposed view: rs=ld, cs=1).
cudaError_t ew_binary(int op, int rows, int cols, const double* a, long long ars, long long acs, const double* b,
                      long long brs, long long bcs, double* o, long long ors, long long ocs, cudaStream_t st);
cudaError_t ew_binary_f32(int op, int rows, int cols, const float* a, long long ars, long long acs, const float* b,
                          long long brs, long long bcs, float* o, long long ors, long long ocs, cudaStream_t st);
cudaError_t ew_unary(int op, int rows, int cols, const double* a, long long ars, long long acs, double* o,
                     long long ors, long long ocs, double alpha, double beta, cudaStream_t st);
// out (cols x rows, ldo) = in (rows x cols, ldi)^T, both column-major
cudaError_t transpose_f64(const double* in, long long ldi, double* out, long long ldo, int rows, int cols, cudaStream_t st);
cudaError_t transpose_b16(const void* in, long long ldi, void* out, long long ldo, int rows, int cols, cudaStream_t st);
cudaError_t transpose_b32(const void* in, long long ldi, void* out, long long ldo, int rows, int cols, cudaStream_t st);
int sum_scratch_doubles();
cudaError_t sum_f64(const double* a, int rows, int cols, long long ld, double* scratch, cudaStream_t st);
cudaError_t convert_strided(int src_dtype, int dst_dtype, int rows, int cols, const void* a, long long ars,
                            long long acs, void* o, long long ors, long long ocs, cudaStream_t st);
cudaError_t fill_uniform_f64(double* out, long long rs, long long cs, int rows, int cols, int row_major,
                             unsigned long long state0, long long first, double lo, double hi, cudaStream_t st);
// Device address of the generator's jump tables: 40 x 64 words, row j = the columns of T^(2^j) (T = one XORShift step).
cudaError_t fill_jump_tables(const unsigned long long** tables);

}  // namespace mb

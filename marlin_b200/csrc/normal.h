// StandardNormalGenerator (utils/RandomDataGenerator.scala:70-82) on the device: java.util.Random.nextGaussian over the
// XORShift stream of a partition, count, scan and write.  See normal.cu.
#pragma once
#include <cuda_runtime.h>

namespace mb {

// Attempts of the polar method per tile of the count and write passes (MB_NORMAL_TILE_ATTEMPTS).
constexpr int NORMAL_TILE_ATTEMPTS = 32768;

// The first n = rows * cols values of mean + sd * nextGaussian() from XORShift state `state0`, written to
// out[r * rs + c * cs] in fill order (row_major: rows one after another; else column-major).  sd is sqrt(variance),
// already rounded.  Blocking: one stream synchronisation per counting round.  *attempts_used (when not null) receives A,
// the index of the last attempt the values used plus one (one more synchronisation).  cudaErrorInvalidValue when the
// counted attempts would reach beyond `max_positions` nextDouble positions.
cudaError_t fill_normal_f64(double* out, long long rs, long long cs, int rows, int cols, int row_major,
                            unsigned long long state0, double mean, double sd, long long max_positions,
                            long long* attempts_used, cudaStream_t st);

}  // namespace mb

// CoordinateMatrix.ALS (ml/ALSHelp.scala:292-382, updateBlock): the per-entity normal equations of one ALS half-step,
// assembled in the reference's order and solved by Cholesky, and the COO -> dense-row scatter of toDenseVecMatrix.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace mb {

// One side's links on the device.  Position p (an entity of this side, ordered by block then id) has the ratings
// [offsets[p], offsets[p+1]) with the partner's factor row partners[q] of the other side and the rating ratings[q], in
// the reference's term order.  work[0..count) lists the positions to process, heaviest first; ids[p] is the entity id.
struct AlsLinks {
    const int32_t* ids;
    const long long* offsets;
    const int32_t* partners;
    const float* ratings;
    const int32_t* work;
    long long count;
};

// Y: the fixed side's factor rows (row i at Y + i * ldy).  yty (rank x rank, element (i, j) at yty[i * ldyty + j]) is
// added after the regularisation when implicit.  X: the solved rows (position p at X + p * ldx).  A non-positive pivot
// leaves the row unwritten and lowers *bad to the entity's id (*bad starts at INT32_MAX).
cudaError_t als_solve(const AlsLinks& L, int rank, const double* Y, long long ldy, double lambda, double alpha, bool implicit,
                      const double* yty, long long ldyty, double* X, long long ldx, int* bad, cudaStream_t st);
// The same assembly, stopped before the factorisation: packed lower triangle (row-major, rank (rank + 1) / 2 doubles)
// of position p at A + p * tri, b at B + p * rank.
cudaError_t als_assemble(const AlsLinks& L, int rank, const double* Y, long long ldy, double lambda, double alpha,
                         bool implicit, const double* yty, long long ldyty, double* A, double* B, cudaStream_t st);

// out[row[e] * ld + col[e]] = val[e] for e < nnz; no two entries may share (row, col).
cudaError_t coo_scatter_rows(long long nnz, const int32_t* row, const int32_t* col, const float* val, double* out,
                             long long ld, cudaStream_t st);

}  // namespace mb

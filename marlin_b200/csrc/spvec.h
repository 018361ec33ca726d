#pragma once
#include "sparse.h"
#include "stream_buffer.h"

namespace mb {

// Device scratch of one row-wise product, made by spvec_count and used by spvec_fill: the rows of each bin and each row's
// candidate column range.
struct SpvecWork {
    StreamBuffer lists;          // int: bin b's rows at lists[b * rows .. + bins[b])
    StreamBuffer range;          // int2: lowest and highest column any product of the row can reach
    StreamBuffer bin_size;       // int: 3 counters, then the int64 total
    int bins[3] = {0, 0, 0};
};

// C = A * B row by row, A and B CSR (A.cols == B.rows).  spvec_count writes rowptr (A.rows + 1 entries: 0, then the
// inclusive scan of each row's distinct output columns) and the total into *total (may exceed 2^31 - 1, in which case
// rowptr is not usable).  It synchronises the stream twice, to read the bin sizes and the total.
cudaError_t spvec_count(const CsrView& A, const CsrView& B, int* rowptr, long long* total, SpvecWork* w, cudaStream_t st);
// The numeric pass: colidx / vals (rowptr[A.rows] entries) get each row's columns ascending and the float32 sums widened
// to double.
cudaError_t spvec_fill(const CsrView& A, const CsrView& B, const SpvecWork& w, const int* rowptr, int* colidx, double* vals,
                       cudaStream_t st);

// Row-major dense rows (rows x cols view D) -> CSR keeping v != 0.0.  The count pass writes rowptr (rows + 1) and *total
// (one stream synchronisation); the compact pass fills colidx / vals.
cudaError_t dense_rows_count(DView D, int rows, int cols, int* rowptr, long long* total, cudaStream_t st);
cudaError_t dense_rows_compact(DView D, int rows, int cols, const int* rowptr, int* colidx, double* vals, cudaStream_t st);

// rowptr[r] = r * s for r <= rows, and rows 1 .. rows-1 of colidx take a copy of row 0's s columns.
cudaError_t spvec_replicate_columns(int rows, int s, int* rowptr, int* colidx, cudaStream_t st);

}  // namespace mb

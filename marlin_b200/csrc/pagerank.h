#pragma once
#include "sparse.h"

namespace mb {

// The rows of an in-link CSR (nnz entries) whose in-degree exceeds MB_PAGERANK_LIGHT_BOUND, found once per matrix by
// pagerank_plan (one stream synchronisation to read their count) and read by every pagerank_step.  p->heavy is a
// cudaMalloc allocation the caller frees with cudaFree, also when the call fails.
struct PagerankPlan {
    int* heavy = nullptr;        // heavy row ids, then the counter
    int nheavy = 0;
};
cudaError_t pagerank_plan(const CsrView& L, long long nnz, PagerankPlan* p, cudaStream_t st);

// y_i = fl(fl(P_0 + P_1 + ...) + addend) for every row i of L (rows = targets, colidx = ascending sources), P_s the
// sequential sum from 0.0 of fl(w * x_j) over the row's sources j in [s * seg_len, (s + 1) * seg_len).  x has L.cols
// elements, y L.rows; y must not overlap x.  Two launches (light rows, heavy rows); no synchronisation.
cudaError_t pagerank_step(const CsrView& L, const PagerankPlan& p, const double* x, long long seg_len, double addend,
                          double* y, cudaStream_t st);

}  // namespace mb

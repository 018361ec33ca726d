// The NeuralNetwork example (examples/NeuralNetwork.scala): everything of one mini-batch iteration of the two-layer sigmoid
// network that is not one of the two large GEMMs -- the output layer, both deltas, the output-weight gradient and the
// weight update.
#pragma once
#include <cuda_runtime.h>
#include <cstddef>

namespace mb {

constexpr int NN_CLASSES = 10;          // columns of the output weight (BDM.rand(layerNum, 10), :206)
constexpr int NN_RESIDENT_H = 512;      // widest hidden layer whose row tile and output weight stay in shared memory

// Number of per-CTA partials nn_backprop_f64 writes for a block of r rows (its grid size).
int nn_parts(int r, int num_sms);

// One block of the selection, after hiddenLayerInput Z1 = X W1 (:222-225) has been formed:
//   A1 = sigmoid(Z1), Z2 = A1 W2, A2 = sigmoid(Z2)                       (:226-231)
//   D2 = (1 - A2) A2 (A2 - onehot(labels))                               (:119-128, :152-162)
//   D1 = (1 - A1) A1 (D2 W2^T)                                           (:240-241)
//   part[p] (H x 10, column-major, packed) = the rows of CTA p's tiles of A1^T D2, in ascending row order
// z1: r x H column-major, ld >= r, 8-byte aligned.  d1 (r x H, ldd) may be z1 itself: the block is then replaced in place.
// w2: H x 10 column-major with leading dimension ldw2.  labels: r device ints in [0, 10).  part: nn_parts(r, num_sms) * H * 10
// doubles.  A1, Z2, A2 and D2 never reach device memory.  For H <= NN_RESIDENT_H z1 is read once; wider layers are read a
// second time for D1.  Deterministic: the same inputs give the same bits on every run.  One launch.
cudaError_t nn_backprop_f64(const double* z1, long long ld, int r, int H, const double* w2, long long ldw2, const int* labels,
                            double* d1, long long ldd, double* part, int num_sms, cudaStream_t st);

// For each element (i, j) of a rows x cols weight: s = sum over blocks b (ascending) of
//   fl(scale * (part[first[b]] + part[first[b] + 1] + ... + part[first[b + 1] - 1])(i, j)),
// the way computeWeightUpd scales each block's product before the sum (:171-183); then out(i, j) = s, or, when out is null,
// w(i, j) -= s.  part p is rows x cols with leading dimension ldp at part + p * stride; first: nblocks + 1 device ints.
cudaError_t nn_apply_f64(const double* part, long long ldp, long long stride, const int* first, int nblocks, int rows, int cols,
                         double scale, double* out, long long ldo, double* w, long long ldw, cudaStream_t st);

}  // namespace mb

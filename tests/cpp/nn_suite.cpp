// The NeuralNetwork example through the compiled host mirror (include/marlin_b200.hpp): one step of a case worked by hand,
// and the errors.  Exits 3 without a GPU (there is no CPU fallback), 1 on a failed check.
//
// Rows [a, a] against W1 = [[1, 2], [-1, -2]] give Z1 = 0 and W2 = [v; -v] gives Z2 = 0, so every sigmoid is 0.5:
// D2(r, j) = 0.125 (-0.125 at the label), E1(r, h) = s_h t_r with s = (1, -1) and t_r = 0.125 (sum(v) - 2 v[y_r]),
// D1 = 0.25 E1.  Every product and sum below is exact in binary floating point.
#include "marlin_b200.hpp"
#include "suite.h"

#include <cstdio>

using namespace marlin;

int main() {
    if (!require_gpu()) return 3;
    DenseMatrix W1{{1.0, 2.0}, {-1.0, -2.0}}, W2(2, 10);
    double vsum = 0.0;
    for (int j = 0; j < 10; ++j) { W2(0, j) = j + 1.0; W2(1, j) = -(j + 1.0); vsum += j + 1.0; }
    const std::vector<std::vector<double>> a{{1.0, 2.0, 4.0}, {8.0}};
    const std::vector<std::vector<int32_t>> y{{0, 3, 3}, {9}};
    examples::NeuralNetwork net(W1, W2);
    for (size_t b = 0; b < a.size(); ++b) {
        DenseMatrix X((int)a[b].size(), 2);
        for (size_t r = 0; r < a[b].size(); ++r) X((int)r, 0) = X((int)r, 1) = a[b][r];
        CHECK(net.addBlock(X, y[b]) == (int)b);
    }
    net.step({0, 1}, 1.0, 4);                                   // learningRate / batchSize = 0.25
    double g1 = 0.0;                                            // dW1(i, h) = s_h * g1
    int count[10] = {};
    for (size_t b = 0; b < a.size(); ++b) {
        double blk = 0.0;
        for (size_t r = 0; r < a[b].size(); ++r) {
            blk += a[b][r] * 0.25 * (0.125 * (vsum - 2.0 * (y[b][r] + 1.0)));
            ++count[y[b][r]];
        }
        g1 += 0.25 * blk;
    }
    const DenseMatrix h = net.hiddenWeight(), o = net.outputWeight();
    CHECK(g1 != 0.0);
    for (int i = 0; i < 2; ++i) {
        CHECK(h(i, 0) == W1(i, 0) - g1 && h(i, 1) == W1(i, 1) + g1);
        for (int j = 0; j < 10; ++j) CHECK(o(i, j) == W2(i, j) - 0.25 * 0.5 * 0.125 * (4 - 2.0 * count[j]));
    }
    CHECK(throws([&] { net.addBlock(DenseMatrix(2, 2), {0, 10}); }));           // label out of range
    CHECK(throws([&] { net.addBlock(DenseMatrix(2, 2), {0}); }));               // one label for two rows
    CHECK(throws([&] { net.step({}, 1.0, 4); }));                               // nothing selected
    CHECK(throws([&] { net.step({7}, 1.0, 4); }));                              // no such block
    examples::NeuralNetwork narrow(DenseMatrix(3, 2), W2);
    narrow.addBlock(DenseMatrix(2, 2), {1, 2});
    CHECK(throws([&] { narrow.step({0}, 1.0, 4); }));                           // 2 features against 3 weight rows
    return finish("nn suite");
}

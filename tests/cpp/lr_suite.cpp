// DenseVecMatrix::lr through the compiled host mirror (include/marlin_b200.hpp): one exact first step on dyadic data, a
// 50-step run against a host restatement of :1005-1035, and the empty matrix.  Exits 3 without a GPU (there is no CPU
// fallback), 1 on a failed check.
#include "marlin_b200.hpp"
#include "suite.h"

#include <cmath>
#include <cstdio>
#include <random>

using namespace marlin;

// :1005-1035 on the host, rows in order, no FMA contraction in the expressions that matter (volatile temporaries)
static std::vector<double> host_lr(const std::vector<DenseVecMatrix::Row>& rows, long dataSize, double step, int iters) {
    const size_t n = rows[0].second.size();
    std::vector<double> w(n, 0.0);
    for (int i = 1; i <= iters; ++i) {
        std::vector<double> delta(n, 0.0);
        for (auto& r : rows) {
            volatile double dot = 0.0;
            for (size_t j = 0; j < n; ++j) { volatile double p = (j == 0 ? 1.0 : r.second[j]) * w[j]; dot = dot + p; }
            const double g = 1.0 / (1.0 + std::exp(-1.0 * dot)) - r.second[0];
            for (size_t j = 0; j < n; ++j) { volatile double p = (j == 0 ? 1.0 : r.second[j]) * g; delta[j] = delta[j] + p; }
        }
        const double scale = step / (double)dataSize / std::sqrt((double)i);
        for (size_t j = 0; j < n; ++j) { volatile double p = delta[j] * scale; w[j] = w[j] - p; }
    }
    return w;
}

int main() {
    if (!require_gpu()) return 3;
    // dyadic features, labels 0 / 1, 64 rows: the first step is exact in any summation order
    std::mt19937_64 gen(3);
    std::vector<DenseVecMatrix::Row> rows;
    for (long i = 0; i < 64; ++i) {
        std::vector<double> v(37);
        v[0] = (double)(gen() & 1);
        for (size_t j = 1; j < v.size(); ++j) v[j] = (double)((long)(gen() % 17) - 8) / 4.0;
        rows.emplace_back(i, v);
    }
    DenseVecMatrix mat(rows);
    const std::vector<double> one = mat.lr(1.0, 1), want1 = host_lr(rows, 64, 1.0, 1);
    CHECK(one.size() == 37);
    for (size_t j = 0; j < one.size(); ++j) CHECK(one[j] == want1[j]);
    // 50 steps: exp and the order of the sums may differ in the last bits, so a relative tolerance
    const std::vector<double> fifty = mat.lr(0.5, 50), want50 = host_lr(rows, 64, 0.5, 50);
    double err = 0.0, scale = 0.0;
    for (size_t j = 0; j < fifty.size(); ++j) { err = std::max(err, std::fabs(fifty[j] - want50[j])); scale = std::max(scale, std::fabs(want50[j])); }
    CHECK(err <= 1e-12 * scale);
    CHECK(mat.lr(1.0, 0) == std::vector<double>(37, 0.0));
    // an id gap: dataSize is max id + 1
    std::vector<DenseVecMatrix::Row> gap = {{0, {1.0, 2.0}}, {9, {0.0, -1.0}}};
    DenseVecMatrix g(gap);
    const std::vector<double> gw = g.lr(1.0, 1), gwant = host_lr(gap, 10, 1.0, 1);
    CHECK(gw[0] == gwant[0] && gw[1] == gwant[1]);
    // rows of another width than numCols(): an error, not a w of the wrong size
    CHECK(throws<std::invalid_argument>([&] { DenseVecMatrix(rows, 0, 5).lr(1.0, 1); }));
    // the empty matrix
    CHECK(throws<std::runtime_error>([] { DenseVecMatrix(std::vector<DenseVecMatrix::Row>{}, 0, 0).lr(1.0, 1); }));
    return finish("lr suite");
}

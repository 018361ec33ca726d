// The six-argument DenseVecMatrix::computeSVD of the compiled host mirror (include/marlin_b200.hpp): the Lanczos modes on a
// small tall matrix against the four-argument overload's Gramian and Jacobi path.  Exits 3 without a GPU (there is no
// CPU fallback), 1 on a failed check.
#include "marlin_b200.hpp"
#include "suite.h"

#include <cmath>
#include <cstdio>
#include <random>

using namespace marlin;

int main() {
    if (!require_gpu()) return 3;
    std::mt19937_64 gen(17);
    std::normal_distribution<double> nd;
    std::vector<DenseVecMatrix::Row> tall;
    for (long i = 0; i < 3000; ++i) {
        std::vector<double> v(64);
        for (auto& x : v) x = nd(gen);
        tall.emplace_back(i, v);
    }
    DenseVecMatrix big(tall);
    auto ref = big.computeSVD(8, true, 1e-9, "local-svd");
    for (const char* mode : {"dist-eigs", "local-eigs", "auto"}) {
        auto got = big.computeSVD(8, true, 1e-9, 300, 1e-10, mode);
        CHECK(got.s.size() == 8 && got.V.rows == 64 && got.V.cols == 8 && got.U != nullptr);
        for (int i = 0; i < 8 && i < (int)got.s.size(); ++i) CHECK(std::fabs(got.s[i] - ref.s[i]) <= 1e-10 * ref.s[0]);
        double orth = 0.0;
        for (int i = 0; i < 8; ++i)
            for (int j = 0; j < 8; ++j) {
                double d = 0.0;
                for (int r = 0; r < 64; ++r) d += got.V(r, i) * got.V(r, j);
                orth = std::max(orth, std::fabs(d - (i == j ? 1.0 : 0.0)));
            }
        CHECK(orth <= 1e-10);
    }
    std::string msg;
    try { big.computeSVD(8, false, 1e-9, 0, 1e-10, "dist-eigs"); } catch (const std::invalid_argument& e) { msg = e.what(); }
    CHECK(msg.rfind("ARPACK returns non-zero info = -4", 0) == 0);
    return finish("eigs suite");
}

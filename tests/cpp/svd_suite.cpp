// DenseVecMatrix::computeSVD through the compiled host mirror (include/marlin_b200.hpp): the reference suite's SVD case
// (DistributedMatrixSuite.scala:375-388, commented out there), a tall random matrix against its own Gramian, and the
// reference's argument errors.  Exits 3 without a GPU (there is no CPU fallback), 1 on a failed check.
#include "marlin_b200.hpp"

#include <cmath>
#include <cstdio>
#include <random>

using namespace marlin;

static int failed = 0;
#define CHECK(c) do { if (!(c)) { std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); ++failed; } } while (0)

int main() {
    try {
        Context::get();
    } catch (const std::exception& e) {
        std::printf("cannot initialise marlin_b200: %s\n", e.what());
        return 3;
    }
    const std::vector<DenseVecMatrix::Row> rows = {{0, {2.0, 0.0, 8.0, 6.0, 0.0}}, {1, {1.0, 6.0, 0.0, 1.0, 7.0}},
                                                   {2, {5.0, 0.0, 7.0, 4.0, 0.0}}, {3, {7.0, 0.0, 8.0, 5.0, 0.0}},
                                                   {4, {0.0, 10.0, 0.0, 0.0, 7.0}}};
    DenseVecMatrix mat(rows);
    auto svd = mat.computeSVD(3, true);
    const double want[3] = {17.92, 15.17, 3.56};
    CHECK(svd.s.size() == 3 && svd.V.rows == 5 && svd.V.cols == 3 && svd.U != nullptr);
    for (int i = 0; i < 3 && i < (int)svd.s.size(); ++i) CHECK(std::fabs(std::round(svd.s[i] * 100.0) / 100.0 - want[i]) < 1e-12);
    // U = A V S^-1, row by row
    DenseMatrix u = svd.U->toBreeze();
    double err = 0.0;
    for (int r = 0; r < 5; ++r)
        for (int j = 0; j < 3; ++j) {
            double acc = 0.0;
            for (int c = 0; c < 5; ++c) acc += rows[r].second[c] * svd.V(c, j);
            err = std::max(err, std::fabs(u(r, j) - acc / svd.s[j]));
        }
    CHECK(err <= 1e-12);
    // a tall matrix: V orthonormal, every mode agrees on s
    std::mt19937_64 gen(5);
    std::normal_distribution<double> nd;
    std::vector<DenseVecMatrix::Row> tall;
    for (long i = 0; i < 3000; ++i) {
        std::vector<double> v(64);
        for (auto& x : v) x = nd(gen);
        tall.emplace_back(i, v);
    }
    DenseVecMatrix big(tall);
    auto a = big.computeSVD(8, false, 1e-9, "local-svd");
    auto b = big.computeSVD(8, false, 1e-9, "dist-eigs");
    CHECK(!a.U && a.s.size() == 8 && b.s.size() == 8);
    for (int i = 0; i < 8 && i < (int)a.s.size(); ++i) CHECK(a.s[i] == b.s[i]);
    double orth = 0.0;
    for (int i = 0; i < 8; ++i)
        for (int j = 0; j < 8; ++j) {
            double d = 0.0;
            for (int r = 0; r < 64; ++r) d += a.V(r, i) * a.V(r, j);
            orth = std::max(orth, std::fabs(d - (i == j ? 1.0 : 0.0)));
        }
    CHECK(orth <= 1e-12);
    // the reference's requires
    auto message = [&](int k, const std::string& mode) -> std::string {
        try { mat.computeSVD(k, false, 1e-9, mode); } catch (const std::invalid_argument& e) { return e.what(); }
        return "";
    };
    CHECK(message(0, "auto") == "Request up to n singular values but got k=0 and n=5.");
    CHECK(message(2, "lanczos") == "Do not support mode lanczos.");
    CHECK(message(5, "local-eigs") == "k must be smaller than n in local-eigs mode but got k=5 and n=5.");
    std::printf("svd suite: %d failed checks\n", failed);
    return failed ? 1 : 0;
}

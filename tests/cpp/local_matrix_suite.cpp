// LocalMatrixSuite.scala:8-72 through the compiled host mirror (include/marlin_b200.hpp): the reference's four exact 4x4
// cases (toDense, dense x sparse, sparse x sparse, sparse x dense), plus the sparse SubMatrix dispatch, the scalar ops,
// toDenseBlocks, a sparse BlockMatrix multiply and the sparse generator's checks.  Exits 3 without a GPU (there is no CPU
// fallback), 1 on a failed check.
#include "marlin_b200.hpp"
#include "suite.h"

#include <cstdio>

using namespace marlin;

template <class F> static bool throwsInvalid(F f, const char* needle) {
    try { f(); } catch (const std::invalid_argument& e) { return std::string(e.what()).find(needle) != std::string::npos; }
    return false;
}

int main() {
    if (!require_gpu()) return 3;
    const SparseMatrix spMat(4, 4, {SparseVector(4, {1}, {1.0}), SparseVector(4, {0, 3}, {2.0, 1.0}), SparseVector(4, {0}, {3.0}),
                                    SparseVector(4, {2}, {4.0})});
    const DenseMatrix deMat{{0.0, 1.0, 2.0, 3.0}, {2.0, 3.0, 4.0, 5.0}, {3.0, 2.0, 1.0, 0.0}, {1.0, 1.0, 1.0, 1.0}};
    // "sparse matrix to breeze `DenseMatrix`"
    CHECK((spMat.toDense() == DenseMatrix{{0.0, 2.0, 3.0, 0.0}, {1.0, 0.0, 0.0, 0.0}, {0.0, 0.0, 0.0, 4.0}, {0.0, 1.0, 0.0, 0.0}}));
    // "breeze `DenseMatrix` multiply sparse matrix"
    CHECK((LibMatrixMult::multDenseSparse(deMat, spMat) ==
           DenseMatrix{{1.0, 3.0, 0.0, 8.0}, {3.0, 9.0, 6.0, 16.0}, {2.0, 6.0, 9.0, 4.0}, {1.0, 3.0, 3.0, 4.0}}));
    // "sparse matrix multiply sparse matrix"
    const DenseMatrix ss{{2.0, 0.0, 0.0, 12.0}, {0.0, 2.0, 3.0, 0.0}, {0.0, 4.0, 0.0, 0.0}, {1.0, 0.0, 0.0, 0.0}};
    CHECK(spMat.multiply(spMat) == ss);
    // "sparse matrix multiply breeze `DenseMatrix`"
    const DenseMatrix sd{{13.0, 12.0, 11.0, 10.0}, {0.0, 1.0, 2.0, 3.0}, {4.0, 4.0, 4.0, 4.0}, {2.0, 3.0, 4.0, 5.0}};
    CHECK(LibMatrixMult::multSparseDense(spMat, deMat) == sd);

    // SubMatrix: the four sparsity pairs, the scalar ops (stored values only) and the reference's error message
    SubMatrix S(spMat), D(deMat);
    CHECK(S.isSparse() && !D.isSparse() && S.rows() == 4 && S.cols() == 4 && S.nnz() == 5);
    CHECK(S.multiply(S).denseBlock() == ss && S.multiply(D).denseBlock() == sd);
    CHECK(!S.multiply(D).isSparse());
    SubMatrix plus = S.add(1.0);
    CHECK(plus.isSparse() && plus.nnz() == 5);
    CHECK((plus.denseBlock() == DenseMatrix{{0.0, 3.0, 4.0, 0.0}, {2.0, 0.0, 0.0, 0.0}, {0.0, 0.0, 0.0, 5.0}, {0.0, 2.0, 0.0, 0.0}}));
    CHECK(S.multiply(2.0).sparseBlock().values[1].values == (std::vector<double>{4.0, 2.0}));
    CHECK(S.divide(2.0).sparseBlock().values[3].values == (std::vector<double>{2.0}));
    CHECK(S.subtract(1.0).sparseBlock().values[0].indices == (std::vector<int32_t>{1}));
    CHECK(throwsInvalid([&] { S.add(D); }, "Not supported add-operator between matrices of sparsity with true and false"));
    CHECK(throwsInvalid([&] { SubMatrix bad(SparseMatrix(4, 1, {SparseVector(4, {3, 0}, {1.0, 2.0})})); }, "not strictly increasing"));

    // BlockMatrix: sparse x sparse on a 2 x 2 grid against toDenseBlocks + DMMA, and the generator
    BlockMatrix A = MTUtils::randomBlockMatrix(300, 260, 2, 2, {true, 0.05}, 7);
    BlockMatrix B = MTUtils::randomBlockMatrix(260, 210, 2, 2, {true, 0.05}, 8);
    CHECK(A.hasSparse() && !A.toDenseBlocks().hasSparse());
    const DenseMatrix got = A.multiply(B).toBreeze();
    BlockMatrix Ad = A.toDenseBlocks(), Bd = B.toDenseBlocks();
    const DenseMatrix ref = Ad.multiply(Bd).toBreeze();
    double err = 0.0;
    for (size_t i = 0; i < got.data.size(); ++i) err = std::max(err, std::fabs(got.data[i] - ref.data[i]));
    CHECK(got.rows == 300 && got.cols == 210 && err <= 1e-12);
    for (auto& kv : A.blocks) {
        const SparseMatrix sm = kv.second.sparseBlock();
        const size_t s = (size_t)(sm.numCols * 0.05);
        for (auto& v : sm.values) {
            CHECK(v.indices.size() == s);
            for (size_t t = 1; t < v.indices.size(); ++t) CHECK(v.indices[t] > v.indices[t - 1]);
            for (double x : v.values) CHECK(x >= 0.0 && x < 1.0);
        }
    }
    CHECK(throwsInvalid([] { MTUtils::randomBlockMatrix(10, 200, 1, 1, {true, 0.1}, 1); }, "non-zeros per column asked"));
    CHECK(throwsInvalid([] { MTUtils::randomBlockMatrix(10, 10, 1, 1, {true, 0.0}, 1); }, "must be positive"));
    return finish("local_matrix_suite");
}

// C++ port of the hot-path cases of the reference's DistributedMatrixSuite
// (/root/reference/src/test/scala/edu/nju/pasalab/marlin/matrix/DistributedMatrixSuite.scala), written against the
// compiled host mirror include/marlin_b200.hpp.  Every expected value is the reference's own golden literal (small
// integers, so assertions are exact).  Needs an H100; without one the first call throws the library's
// "no CPU fallback" error and the program exits with status 3.
#include "marlin_b200.hpp"
#include "suite.h"

#include <cstdio>
#include <functional>
#include <iostream>

using namespace marlin;
using BDM = DenseMatrix;

static int passed = 0;
static void test(const char* name, const std::function<void()>& body) {
    const int before = failed;
    try { body(); } catch (const std::exception& e) { std::printf("  EXCEPTION in '%s': %s\n", name, e.what()); ++failed; }
    if (failed == before) ++passed;
    std::printf("[%s] %s\n", failed == before ? " ok " : "FAIL", name);
}

// DMS.scala:15-24 — the shared fixture: rows deliberately out of order; the same matrix as a 2x2 grid of 2x2 blocks
static std::vector<DenseVecMatrix::Row> data() {
    return {{0, {0.0, 1.0, 2.0, 3.0}}, {2, {3.0, 2.0, 1.0, 0.0}}, {3, {1.0, 1.0, 1.0, 1.0}}, {1, {2.0, 3.0, 4.0, 5.0}}};
}
static BlockMatrix::Blocks blks() {
    return {{BlockID(0, 0), SubMatrix(BDM{{0.0, 1.0}, {2.0, 3.0}})}, {BlockID(0, 1), SubMatrix(BDM{{2.0, 3.0}, {4.0, 5.0}})},
            {BlockID(1, 0), SubMatrix(BDM{{3.0, 2.0}, {1.0, 1.0}})}, {BlockID(1, 1), SubMatrix(BDM{{1.0, 0.0}, {1.0, 1.0}})}};
}
static bool contains(BlockMatrix& m, BlockID id, const BDM& expected) {
    for (auto& kv : m.blocks)
        if (kv.first == id && kv.second.denseBlock() == expected) return true;
    return false;
}

int main() {
    if (!require_gpu()) return 3;
    const BDM expectedDense{{0.0, 1.0, 2.0, 3.0}, {2.0, 3.0, 4.0, 5.0}, {3.0, 2.0, 1.0, 0.0}, {1.0, 1.0, 1.0, 1.0}};
    const BDM expectedProduct{{11.0, 10.0, 9.0, 8.0}, {23.0, 24.0, 25.0, 26.0}, {7.0, 11.0, 15.0, 19.0}, {6.0, 7.0, 8.0, 9.0}};

    test("matrix size", [&] {                                                     // :42-51
        DenseVecMatrix mat(data());
        CHECK(mat.numRows() == 4 && mat.numCols() == 4);
        BlockMatrix ma(blks());
        CHECK(ma.numRows() == 4 && ma.numCols() == 4 && ma.numBlksByRow() == 2 && ma.numBlksByCol() == 2);
    });
    test("empty rows", [&] {                                                      // :53-71
        DenseVecMatrix mat(std::vector<DenseVecMatrix::Row>{});
        CHECK(throws<std::runtime_error>([&] { mat.numRows(); }));
        CHECK(throws<std::runtime_error>([&] { mat.numCols(); }));
        BlockMatrix ma(BlockMatrix::Blocks{});
        CHECK(throws<std::runtime_error>([&] { ma.numRows(); }));
        CHECK(throws<std::runtime_error>([&] { ma.numCols(); }));
    });
    test("to Breeze local Matrix", [&] {                                          // :73-84
        DenseVecMatrix mat(data());
        CHECK(mat.toBreeze() == expectedDense);
        BlockMatrix ma(blks());
        CHECK(ma.toBreeze() == expectedDense);
    });
    test("to BlockMatrix", [&] {                                                  // :86-105
        DenseVecMatrix mat(data());
        BlockMatrix blkMat = mat.toBlockMatrix(2, 2);
        CHECK(mat.numRows() == blkMat.numRows() && mat.numCols() == blkMat.numCols());
        CHECK(contains(blkMat, BlockID(0, 0), BDM{{0.0, 1.0}, {2.0, 3.0}}));
        CHECK(contains(blkMat, BlockID(0, 1), BDM{{2.0, 3.0}, {4.0, 5.0}}));
        CHECK(contains(blkMat, BlockID(1, 0), BDM{{3.0, 2.0}, {1.0, 1.0}}));
        CHECK(contains(blkMat, BlockID(1, 1), BDM{{1.0, 0.0}, {1.0, 1.0}}));
        BlockMatrix blkMat2 = mat.toBlockMatrix(1, 4);
        CHECK(blkMat.toBreeze() == expectedDense && blkMat2.toBreeze() == expectedDense);
    });
    test("to DenseVecMatrix", [&] {                                               // :108-119
        BlockMatrix ma(blks());
        DenseVecMatrix d = ma.toDenseVecMatrix();
        CHECK(ma.numRows() == d.numRows() && ma.numCols() == d.numCols());
        CHECK(d.toBreeze() == expectedDense);
    });
    test("Matrix-matrix and element-wise addition/subtract; element-wise multiply and divide", [&] {   // :164-205
        const BDM eleAdd1{{1.0, 2.0, 3.0, 4.0}, {3.0, 4.0, 5.0, 6.0}, {4.0, 3.0, 2.0, 1.0}, {2.0, 2.0, 2.0, 2.0}};
        const BDM addSelf{{0.0, 2.0, 4.0, 6.0}, {4.0, 6.0, 8.0, 10.0}, {6.0, 4.0, 2.0, 0.0}, {2.0, 2.0, 2.0, 2.0}};
        const BDM eleSubtract1{{-1.0, 0.0, 1.0, 2.0}, {1.0, 2.0, 3.0, 4.0}, {2.0, 1.0, 0.0, -1.0}, {0.0, 0.0, 0.0, 0.0}};
        const BDM divide2{{0.0, 0.5, 1.0, 1.5}, {1.0, 1.5, 2.0, 2.5}, {1.5, 1.0, 0.5, 0.0}, {0.5, 0.5, 0.5, 0.5}};
        const BDM zeros(4, 4);
        DenseVecMatrix mat(data());
        CHECK(mat.add(1).toBreeze() == eleAdd1);
        CHECK(mat.add(mat).toBreeze() == addSelf);
        CHECK(mat.subtract(1).toBreeze() == eleSubtract1);
        CHECK(mat.subtract(mat).toBreeze() == zeros);
        CHECK(mat.multiply(2.0).toBreeze() == addSelf);
        CHECK(mat.divide(2).toBreeze() == divide2);
        BlockMatrix ma(blks());
        CHECK(ma.add(1).toBreeze() == eleAdd1);
        CHECK(ma.add(ma).toBreeze() == addSelf);
        CHECK(ma.add(mat).toBreeze() == addSelf);
        CHECK(ma.subtract(1).toBreeze() == eleSubtract1);
        CHECK(ma.subtract(ma).toBreeze() == zeros);
        CHECK(ma.subtract(mat).toBreeze() == zeros);
        CHECK(ma.multiply(2.0).toBreeze() == addSelf);
        CHECK(ma.divide(2).toBreeze() == divide2);
    });
    test("DenseVecMatrix multiply a DenseVecMatrix, and select broadcast-approach", [&] {             // :225-234
        DenseVecMatrix mat(data());
        CHECK(mat.multiply(mat, 2) == expectedProduct);
    });
    test("new matrix multiplication", [&] {                                       // :236-249
        DenseVecMatrix mat(data());
        CHECK(mat.multiply(mat, std::make_tuple(2, 2, 1)).toBreeze() == expectedProduct);
        CHECK(mat.multiply(mat, std::make_tuple(2, 1, 2)).toBreeze() == expectedProduct);
        CHECK(mat.multiply(mat, std::make_tuple(2, 2, 2)).toBreeze() == expectedProduct);
    });
    test("DenseVecMatrix multiply a local matrix", [&] {                          // :251-267
        DenseVecMatrix mat(data());
        CHECK(mat.multiply(expectedDense).toBreeze() == expectedProduct);
        CHECK(mat.multiply(expectedDense).toBreeze() == expectedProduct);
    });
    test("multiply a BlockMatrix", [&] {                                          // :269-287
        DenseVecMatrix mat(data());
        BlockMatrix blkMat(blks());
        CHECK(mat.multiply(blkMat, 2) == expectedProduct);
        BlockMatrix ma(blks());
        BlockMatrix result2 = ma.multiply(ma);
        CHECK(contains(result2, BlockID(0, 0), BDM{{11.0, 10.0}, {23.0, 24.0}}));
        CHECK(contains(result2, BlockID(0, 1), BDM{{9.0, 8.0}, {25.0, 26.0}}));
        CHECK(contains(result2, BlockID(1, 0), BDM{{7.0, 11.0}, {6.0, 7.0}}));
        CHECK(contains(result2, BlockID(1, 1), BDM{{15.0, 19.0}, {8.0, 9.0}}));
    });
    test("BlockMatrix multiply a DenseVecMatrix and choose to run broadcast", [&] {                   // :289-299
        BlockMatrix ma(blks());
        DenseVecMatrix denVecMat(data());
        CHECK(ma.multiply(denVecMat, 2).toBreeze() == expectedProduct);
    });
    test("transpose", [&] {                                                       // :302-316
        DenseVecMatrix mat(data());
        BlockMatrix result = mat.transpose();
        CHECK(contains(result, BlockID(0, 0), BDM{{0.0, 2.0}, {1.0, 3.0}, {2.0, 4.0}, {3.0, 5.0}}));
        CHECK(contains(result, BlockID(0, 1), BDM{{3.0, 1.0}, {2.0, 1.0}, {1.0, 1.0}, {0.0, 1.0}}));
        BlockMatrix ma(blks());
        BlockMatrix result2 = ma.transpose();
        CHECK(contains(result2, BlockID(0, 0), BDM{{0.0, 2.0}, {1.0, 3.0}}));
        CHECK(contains(result2, BlockID(0, 1), BDM{{3.0, 1.0}, {2.0, 1.0}}));
        CHECK(contains(result2, BlockID(1, 0), BDM{{2.0, 4.0}, {3.0, 5.0}}));
        CHECK(contains(result2, BlockID(1, 1), BDM{{1.0, 1.0}, {0.0, 1.0}}));
    });
    test("sum", [&] {                                                             // :319-324
        DenseVecMatrix mat(data());
        BlockMatrix blkMat(blks());
        CHECK(mat.sum() == 30.0);
        CHECK(blkMat.sum() == 30.0);
    });
    test("dot product", [&] {                                                     // :326-338
        const BDM dot{{0.0, 1.0, 4.0, 9.0}, {4.0, 9.0, 16.0, 25.0}, {9.0, 4.0, 1.0, 0.0}, {1.0, 1.0, 1.0, 1.0}};
        DenseVecMatrix mat(data());
        BlockMatrix blkMat(blks());
        CHECK(mat.dotProduct(mat).toBreeze() == dot);
        CHECK(mat.dotProduct(blkMat).toBreeze() == dot);
        CHECK(blkMat.dotProduct(blkMat).toBreeze() == dot);
    });
    test("DenseVecMatrix inverse", [&] {                                           // :340-352
        DenseVecMatrix mat({{0, {0.0, 0.0, 1.0}}, {1, {0.0, 1.0, 0.0}}, {2, {1.0, 0.0, 0.0}}});
        BlockMatrix inv = mat.inverse();
        CHECK(inv.toBreeze() == (BDM{{0.0, 0.0, 1.0}, {0.0, 1.0, 0.0}, {1.0, 0.0, 0.0}}));
        // LU and Cholesky of small exact cases: P A = L U with integer factors, L L^T = A
        DenseVecMatrix a({{0, {2.0, 1.0}}, {1, {4.0, 5.0}}});
        auto lu = a.luDecompose("breeze");
        CHECK(lu.second == (std::vector<int>{1, 0}));                             // pivot: |4| > |2|
        CHECK(lu.first.toBreeze() == (BDM{{4.0, 5.0}, {0.5, -1.5}}));
        DenseVecMatrix spd({{0, {4.0, 2.0}}, {1, {2.0, 10.0}}});
        CHECK(spd.choleskyDecompose().toBreeze() == (BDM{{2.0, 0.0}, {1.0, 3.0}}));
        CHECK((throws<std::invalid_argument>([&] { DenseVecMatrix r({{0, {1.0, 2.0, 3.0}}}); r.inverse(); })));
    });

    test("BlockMatrix to BlockMatrix", [&] {                                      // :411-418
        DenseVecMatrix mat(data());
        BlockMatrix blk1 = mat.toBlockMatrix(2, 2);
        CHECK(blk1.toBlockMatrix(1, 4).toBreeze() == blk1.toBreeze());
        CHECK(blk1.toBlockMatrix(4, 1).toBreeze() == blk1.toBreeze());
    });
    test("BlockMatrix multiply a BlockMatrix", [&] {                              // :420-432
        DenseVecMatrix mat(data());
        BlockMatrix blk1 = mat.toBlockMatrix(2, 2);
        BlockMatrix blk2 = mat.toBlockMatrix(1, 4);
        BlockMatrix m = blk1.toBlockMatrix(2, 1);
        CHECK(m.multiply(blk2).toBreeze() == expectedProduct);
    });
    test("BlockMatrix multiply a broadcast matrix", [&] {                         // :434-448
        BlockMatrix blkMat(blks());
        CHECK(blkMat.multiply(expectedDense).toBreeze() == expectedProduct);
    });
    test("disVec to disVec", [&] {                                                // :121-143
        DistributedVector disVec1(std::vector<std::pair<int, std::vector<double>>>{
            {0, {0.0, 1.0, 2.0, 3.0}}, {1, {4.0, 5.0, 6.0, 7.0}}, {2, {8.0, 9.0, 10.0, 11.0}}});
        DistributedVector::SplitStatus splitStatus = {
            {{0, {0, 2}, {0, 2}}, {1, {3, 3}, {0, 0}}},
            {{1, {0, 1}, {1, 2}}, {2, {2, 3}, {0, 1}}},
            {{2, {0, 0}, {2, 2}}, {3, {1, 3}, {0, 2}}}};
        DistributedVector disVec2 = disVec1.toDisVector(splitStatus, 4);
        CHECK(disVec2.splitNum() == 4);
        CHECK(disVec1.toBreeze() == disVec2.toBreeze());
    });
    test("BLAS1 distributed vector multiplication", [&] {                         // :390-409
        std::vector<std::pair<int, std::vector<double>>> vectors = {{0, {1.0, 2.0}}, {1, {3.0, 4.0}}};
        DistributedVector disVec1(vectors), disVec2(vectors);
        const BDM expected{{1.0, 2.0, 3.0, 4.0}, {2.0, 4.0, 6.0, 8.0}, {3.0, 6.0, 9.0, 12.0}, {4.0, 8.0, 12.0, 16.0}};
        DistributedVector t2 = disVec2.transpose(), t1 = disVec1.transpose();
        auto matResult = disVec1.multiply(t2);
        auto doubleResult = t1.multiply(disVec2);
        auto doubleResultLocal = t1.multiply(disVec2, "local");
        CHECK(!matResult.isLeft && matResult.right->toBreeze() == expected);
        CHECK(doubleResult.isLeft && doubleResult.left == 30.0);
        CHECK(doubleResultLocal.isLeft && doubleResultLocal.left == 30.0);
        CHECK(throws<std::invalid_argument>([&] { disVec1.multiply(disVec2); }));
    });
    test("matrix multiply a distributed / broadcast vector", [&] {                // BlockMatrix.scala:240-274
        BlockMatrix ma(blks());
        const std::vector<double> x = {1.0, 2.0, 3.0, 4.0}, y = {20.0, 40.0, 10.0, 10.0};
        DistributedVector dv = DistributedVector::fromVector(x, 2);
        CHECK(ma.multiply(dv).toBreeze() == y);
        DenseVecMatrix mat(data());
        BlockMatrix tall = mat.toBlockMatrix(2, 1);
        CHECK(tall.multiply(x).toBreeze() == y);
        CHECK(throws<std::invalid_argument>([&] { ma.multiply(x); }));
        CHECK(mat.multiply(x) == y);                                              // DenseVecMatrix.scala:171-184
        CHECK(mat.multiply(x, 2).toBreeze() == y);                                // :162-165
        CHECK(mat.multiply(dv, std::make_pair(2, 2)).toBreeze() == y);            // :149-154
    });
    // beyond the reference suite: error behaviour and the generators
    test("dimension mismatch is an IllegalArgumentException", [&] {               // BlockMatrix.scala:150-151, DenseVecMatrix.scala:199-200
        DenseVecMatrix a({{0, {1.0, 2.0, 3.0}}, {1, {4.0, 5.0, 6.0}}});
        CHECK(throws<std::invalid_argument>([&] { a.multiply(a, 2); }));
        BlockMatrix b = a.toBlockMatrix(1, 1);
        CHECK(throws<std::invalid_argument>([&] { b.multiply(b); }));
    });
    test("splitMethod and random generators", [&] {                               // MTUtils.scala:150-175, :34-73
        CHECK(MTUtils::splitMethod(16384, 16384, 16384, 8) == std::make_tuple(2, 2, 2));
        DenseVecMatrix r = MTUtils::randomDenVecMatrix(37, 11, 4, 2024);
        BDM v = r.toBreeze();
        bool inRange = true;
        for (double x : v.data) inRange = inRange && x >= 0.0 && x < 1.0;
        CHECK(v.rows == 37 && v.cols == 11 && inRange);
        BlockMatrix rb = MTUtils::randomBlockMatrix(23, 17, 3, 2, 7);
        CHECK(rb.numBlksByRow() == 3 && rb.numBlksByCol() == 2 && rb.toBreeze().rows == 23);
        BlockMatrix p = rb.transpose();
        CHECK(p.transpose().toBreeze() == rb.toBreeze());
    });

    std::printf("%d tests passed\n", passed);
    return finish("dms suite");
}

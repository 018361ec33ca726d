// C++ port of the reference DistributedMatrixSuite's "slice the matrix" (:207-223) and "repeat by row and column"
// (:354-374) cases, plus cBind, elementMultiply, zeros / ones and norm, written against the compiled host mirror
// include/marlin_b200.hpp.  Every expected value is a small integer, so assertions are exact.  Needs an H100; without one
// the first call throws the library's "no CPU fallback" error and the program exits with status 3.
#include "marlin_b200.hpp"
#include "suite.h"

#include <cmath>
#include <cstdio>
#include <functional>
#include <iostream>

using namespace marlin;
using BDM = DenseMatrix;

template <class F>
static std::string invalidArgument(F f) {
    try { f(); } catch (const std::invalid_argument& e) { return e.what(); } catch (...) { return "<other exception>"; }
    return "<no exception>";
}
static int passed = 0;
static void test(const char* name, const std::function<void()>& body) {
    const int before = failed;
    try { body(); } catch (const std::exception& e) { std::printf("  EXCEPTION in '%s': %s\n", name, e.what()); ++failed; }
    if (failed == before) ++passed;
    std::printf("[%s] %s\n", failed == before ? " ok " : "FAIL", name);
}

// DMS.scala:15-19 — rows deliberately out of order
static std::vector<DenseVecMatrix::Row> data() {
    return {{0, {0.0, 1.0, 2.0, 3.0}}, {2, {3.0, 2.0, 1.0, 0.0}}, {3, {1.0, 1.0, 1.0, 1.0}}, {1, {2.0, 3.0, 4.0, 5.0}}};
}
// a rows x cols matrix of small integers, a(r, c) = (r * 7 + c * 3) % 11 - 5
static BDM ints(int rows, int cols) {
    BDM m(rows, cols);
    for (int r = 0; r < rows; ++r)
        for (int c = 0; c < cols; ++c) m(r, c) = (double)((r * 7 + c * 3) % 11 - 5);
    return m;
}
static DenseVecMatrix rowsOf(const BDM& m) {
    std::vector<DenseVecMatrix::Row> rows;
    for (int r = m.rows - 1; r >= 0; --r) {                                      // out of order on purpose
        std::vector<double> v(m.cols);
        for (int c = 0; c < m.cols; ++c) v[c] = m(r, c);
        rows.push_back({r, v});
    }
    return DenseVecMatrix(rows, m.rows, m.cols);
}
static BDM hstack(const BDM& a, const BDM& b) {
    BDM m(a.rows, a.cols + b.cols);
    for (int r = 0; r < a.rows; ++r) {
        for (int c = 0; c < a.cols; ++c) m(r, c) = a(r, c);
        for (int c = 0; c < b.cols; ++c) m(r, a.cols + c) = b(r, c);
    }
    return m;
}
static BDM tile(const BDM& a, int down, int across) {
    BDM m(a.rows * down, a.cols * across);
    for (int r = 0; r < m.rows; ++r)
        for (int c = 0; c < m.cols; ++c) m(r, c) = a(r % a.rows, c % a.cols);
    return m;
}

int main() {
    if (!require_gpu()) return 3;
    const BDM dense{{0.0, 1.0, 2.0, 3.0}, {2.0, 3.0, 4.0, 5.0}, {3.0, 2.0, 1.0, 0.0}, {1.0, 1.0, 1.0, 1.0}};

    test("slice the matrix", [&] {                                                // :207-223
        DenseVecMatrix mat(data());
        CHECK(mat.sliceByRow(1, 2).toBreeze() == (BDM{{2.0, 3.0, 4.0, 5.0}, {3.0, 2.0, 1.0, 0.0}}));
        CHECK(mat.sliceByColumn(1, 2).toBreeze() == (BDM{{1.0, 2.0}, {3.0, 4.0}, {2.0, 1.0}, {1.0, 1.0}}));
        CHECK(mat.getSubMatrix(1, 2, 1, 2).toBreeze() == (BDM{{3.0, 4.0}, {2.0, 1.0}}));
    });

    test("repeat by row and column", [&] {                                        // :354-374
        DenseVecMatrix mat(data());
        CHECK(MTUtils::repeatByRow(mat, 2).toBreeze() == tile(dense, 1, 2));
        CHECK(MTUtils::repeatByColumn(mat, 2).toBreeze() == tile(dense, 2, 1));
    });

    test("slice requires", [&] {
        DenseVecMatrix mat(data());
        CHECK(invalidArgument([&] { mat.sliceByRow(1, 4); }) == "start row or end row mismatch the matrix num of rows");
        CHECK(invalidArgument([&] { mat.sliceByRow(2, 1); }) == "start row or end row mismatch the matrix num of rows");
        CHECK(invalidArgument([&] { mat.sliceByColumn(0, 4); }) == "start column or end column mismatch the matrix num of columns");
        CHECK(invalidArgument([&] { mat.getSubMatrix(0, 4, 0, 1); }) == "start row or end row dismatch the matrix num of rows");
        CHECK(invalidArgument([&] { mat.getSubMatrix(0, 1, 2, 1); }) == "start column or end column dismatch the matrix num of columns");
        CHECK(invalidArgument([&] { MTUtils::repeatByRow(mat, 0); }) == "repeat times: 0 illegal");
    });

    test("cBind of rows and blocks", [&] {
        const BDM a = ints(9, 5), b = ints(9, 4);
        DenseVecMatrix x = rowsOf(a), y = rowsOf(b);
        CHECK(x.cBind(y).toBreeze() == hstack(a, b));
        BlockMatrix yb = y.toBlockMatrix(2, 2);
        CHECK(x.cBind(yb).toBreeze() == hstack(a, b));
        // widths 3,2 + 2,2 are not the ceil grid of 9 in 4 blocks: the rows route
        BlockMatrix xb = x.toBlockMatrix(2, 2);
        auto r = xb.cBind(yb);
        CHECK(std::holds_alternative<DenseVecMatrix>(r) && std::get<DenseVecMatrix>(r).toBreeze() == hstack(a, b));
        // widths 2,2 + 2,2: relabelled in place
        const BDM c = ints(9, 4);
        BlockMatrix cb = rowsOf(c).toBlockMatrix(3, 2), db = rowsOf(b).toBlockMatrix(3, 2);
        auto s = cb.cBind(db);
        CHECK(std::holds_alternative<BlockMatrix>(s));
        if (std::holds_alternative<BlockMatrix>(s)) {
            BlockMatrix& sb = std::get<BlockMatrix>(s);
            CHECK(sb.numBlksByCol() == 4 && sb.numCols() == 8 && sb.toBreeze() == hstack(c, b));
        }
        CHECK(cb.cBind(y).toBreeze() == hstack(c, b));
        DenseVecMatrix five = rowsOf(ints(5, 4));
        CHECK(invalidArgument([&] { x.cBind(five); }) == "Dimension mismatch:  9 vs 5");
        BlockMatrix fiveb = five.toBlockMatrix(2, 2);
        CHECK(invalidArgument([&] { xb.cBind(fiveb); }) == "Row dimension mismatches: 9 vs 5");
    });

    test("cBind is an inner join", [&] {
        DenseVecMatrix x(data());
        DenseVecMatrix y(std::vector<DenseVecMatrix::Row>{{0, {9.0}}, {3, {8.0}}}, 4, 1);
        DenseVecMatrix r = x.cBind(y);
        CHECK(r.rowIds().size() == 2 && r.numCols() == 5);
        CHECK(r.toBreeze() == (BDM{{0.0, 1.0, 2.0, 3.0, 9.0}, {0.0, 0.0, 0.0, 0.0, 0.0}, {0.0, 0.0, 0.0, 0.0, 0.0}, {1.0, 1.0, 1.0, 1.0, 8.0}}));
    });

    test("repeat on blocks", [&] {
        for (int times = 1; times <= 3; ++times) {
            for (auto shape : {std::make_pair(8, 6), std::make_pair(4, 5)}) {                // widths 3,3 relabel; 3,2 the rows route
                const BDM a = ints(shape.first, shape.second);
                BlockMatrix bm = rowsOf(a).toBlockMatrix(2, 2);
                BlockMatrix r = MTUtils::repeatByRow(bm, times), c = MTUtils::repeatByColumn(bm, times);
                CHECK(r.numCols() == (long)shape.second * times && r.toBreeze() == tile(a, 1, times));
                CHECK(c.numRows() == (long)shape.first * times && c.toBreeze() == tile(a, times, 1));
            }
        }
    });

    test("elementMultiply", [&] {
        const BDM a = ints(6, 5), b = ints(5, 6);
        BDM bt(6, 5), want(6, 5);
        for (int r = 0; r < 6; ++r)
            for (int c = 0; c < 5; ++c) { bt(r, c) = b(c, r); want(r, c) = a(r, c) * b(c, r); }
        BlockMatrix x = rowsOf(a).toBlockMatrix(2, 2), y = rowsOf(bt).toBlockMatrix(2, 2);
        CHECK(x.elementMultiply(y).toBreeze() == want);
        CHECK(x.elementMultiply(y, 0).toBreeze() == want);
        CHECK(x.toBreeze() == a);                                                   // this matrix is unchanged
    });

    test("zeros and ones", [&] {
        CHECK(MTUtils::zerosDenVecMatrix(7, 3).toBreeze() == BDM(7, 3));
        BDM ones(7, 3);
        for (double& v : ones.data) v = 1.0;
        CHECK(MTUtils::onesDenVecMatrix(7, 3).toBreeze() == ones);
    });

    test("norm", [&] {
        DenseVecMatrix mat(data());
        CHECK(mat.norm("1") == 9.0 && mat.norm("inf") == 14.0 && mat.norm("fro") == std::sqrt(86.0));
        const BDM a = ints(5000, 37);
        DenseVecMatrix big = rowsOf(a);
        double one = 0.0, inf = 0.0, sq = 0.0;
        for (int c = 0; c < a.cols; ++c) { double s = 0.0; for (int r = 0; r < a.rows; ++r) s += std::fabs(a(r, c)); one = std::max(one, s); }
        for (int r = 0; r < a.rows; ++r) { double s = 0.0; for (int c = 0; c < a.cols; ++c) { s += std::fabs(a(r, c)); sq += a(r, c) * a(r, c); } inf = std::max(inf, s); }
        CHECK(big.norm("1") == one && big.norm("inf") == inf && big.norm("fro") == std::sqrt(sq));
        CHECK(invalidArgument([&] { mat.norm("2"); }) == "Do not support mode 2.");
    });

    std::printf("%d tests passed\n", passed);
    return finish("dms_api suite");
}

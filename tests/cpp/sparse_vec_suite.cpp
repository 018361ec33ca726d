// SparseVecMatrix through the compiled host mirror (include/marlin_b200.hpp): DistributedMatrixSuite's "generate random
// sparse matrix" (:147-150) and "Sparse matrix multiply" (:152-162), toDenseVecMatrix, toSparseVecMatrix and the errors.
// With a path argument it also writes the COO of randomSpaVecMatrix(300, 200, 0.05, 2, seed 5) * randomSpaVecMatrix(200,
// 150, 0.05, 2, seed 6) there ("row col float-bits" per line) for tests/test_cpp_spvec.py to compare with the Python API.
// Exits 3 without a GPU (there is no CPU fallback), 1 on a failed check.
#include "marlin_b200.hpp"
#include "suite.h"

#include <cmath>
#include <cstdio>
#include <cstring>

using namespace marlin;

int main(int argc, char** argv) {
    if (!require_gpu()) return 3;
    // DistributedMatrixSuite.scala:27-32, 152-162
    std::vector<SparseVecMatrix::Row> data = {{0, {1, 3}, {2.0, 3.0}}, {1, {0, 1}, {5.0, 1.0}}, {2, {3}, {2.0}}, {3, {1, 2}, {1.0, 1.0}}};
    SparseVecMatrix sm(data, 4, 4), sm2(data, 4, 4);
    const double want[4][4] = {{10, 5, 3, 0}, {5, 11, 0, 15}, {0, 2, 2, 0}, {5, 1, 0, 2}};
    DenseMatrix got = sm.multiplySparse(sm2).toBreeze();
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) CHECK(got(i, j) == want[i][j]);

    // :147-150
    SparseVecMatrix s = MTUtils::randomSpaVecMatrix(10, 8, 0.3, 2, 11);
    CHECK(s.nRows() == 10 && s.elementsCount() == 10);
    for (const auto& r : s.rows()) CHECK(r.indices.size() == 2 && r.indices[0] < r.indices[1] && r.indices[1] < 8);

    // toDenseVecMatrix: every id in [0, nRows), absent ids zero
    SparseVecMatrix gaps({{3, {0, 2}, {1.5, -2.0}}, {1, {1}, {4.0}}}, 5, 3);
    DenseVecMatrix d = gaps.toDenseVecMatrix();
    DenseMatrix db = d.toBreeze();
    CHECK(d.rowIds().size() == 5 && db.rows == 5 && db(3, 0) == 1.5 && db(3, 2) == -2.0 && db(1, 1) == 4.0 && db(0, 0) == 0.0);
    // toSparseVecMatrix round trip
    SparseVecMatrix back = d.toSparseVecMatrix();
    CHECK(back.elementsCount() == 5);
    long stored = 0;
    for (const auto& r : back.rows()) stored += (long)r.indices.size();
    CHECK(stored == 3);

    // errors
    CHECK(throws([&] { sm.multiplySparse(SparseVecMatrix(data, 5, 4)); }));                     // nCols != other.nRows
    CHECK(throws([&] { SparseVecMatrix({{1, {0}, {1.0}}, {1, {2}, {1.0}}}, 4, 4); }));          // repeated row id
    CHECK(throws([&] { SparseVecMatrix bad({{0, {2, 1}, {1.0, 1.0}}}, 4, 4); bad.multiplySparse(sm2); }));   // unsorted columns
    CHECK(throws([&] { MTUtils::randomSpaVecMatrix(10, 8, 0.0, 2, 1); }));
    CHECK(throws([&] { MTUtils::randomSpaVecMatrix(10, 8, 1.5, 2, 1); }));

    if (argc > 1) {
        SparseVecMatrix A = MTUtils::randomSpaVecMatrix(300, 200, 0.05, 2, 5), B = MTUtils::randomSpaVecMatrix(200, 150, 0.05, 2, 6);
        CoordinateMatrix C = A.multiplySparse(B);
        std::FILE* f = std::fopen(argv[1], "w");
        for (const auto& e : C.entries()) {
            uint32_t bits;
            std::memcpy(&bits, &e.value, 4);
            std::fprintf(f, "%ld %ld %u\n", e.row, e.col, bits);
        }
        std::fclose(f);
    }
    return finish("sparse_vec suite");
}

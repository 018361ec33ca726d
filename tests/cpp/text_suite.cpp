// The host mirror's matrix-file writers (DenseVecMatrix::saveToFileSystem / saveWithDescription,
// BlockMatrix::saveToFileSystem): writes the files of a fixed matrix under argv[1] for tests/test_cpp_text.py to compare
// with the oracle's lines, and checks the errors here.
#include "suite.h"

#include <filesystem>
#include <limits>
#include <string>

using namespace marlin;

// The value at (i, j) of the suite's matrix; tests/test_cpp_text.py builds the same one.
static double value(int i, int j, int cols) {
    const double inf = std::numeric_limits<double>::infinity();
    const double s[] = {0.0, -0.0, 1.0, -2.5, 0.001, 9.999999999999998e-4, 1e7, 5e-324, 1.7976931348623157e308,
                        std::numeric_limits<double>::quiet_NaN(), inf, -inf, 0.1, 123456.789, 1.0 / 3.0};
    return s[(i * cols + j) % 15] * (i % 2 ? -1.0 : 1.0);
}

int main(int argc, char** argv) {
    if (!require_gpu()) return 3;
    if (argc != 2) return 2;
    const std::string dir = argv[1];
    const int cols = 5;
    const long ids[] = {0, 3, 1, 1L << 40, 7, 5, 6};
    std::vector<DenseVecMatrix::Row> rows, dense;
    for (int i = 0; i < 7; ++i) {
        std::vector<double> v;
        for (int j = 0; j < cols; ++j) v.push_back(value(i, j, cols));
        rows.emplace_back(ids[i], v);
        dense.emplace_back(i, v);
    }
    DenseVecMatrix m(rows);
    m.saveWithDescription(dir + "/rows");
    CHECK(std::filesystem::exists(dir + "/rows/part-00000") && std::filesystem::exists(dir + "/rows/_description"));

    DenseVecMatrix d(dense);
    BlockMatrix b = d.toBlockMatrix(2, 2);
    b.saveToFileSystem(dir + "/blocks", "BlockMatrix");
    b.transpose().saveToFileSystem(dir + "/blocks_t", "blockmatrix");
    b.saveToFileSystem(dir + "/blocks_rows");                                  // any other format: the rows file

    DenseVecMatrix(std::vector<DenseVecMatrix::Row>{}).saveToFileSystem(dir + "/empty");
    CHECK(std::filesystem::file_size(dir + "/empty/part-00000") == 0);

    // a part file that cannot be opened is an IOException
    std::filesystem::create_directories(dir + "/bad/part-00000");
    CHECK(throws<std::ios_base::failure>([&] { m.saveToFileSystem(dir + "/bad"); }));
    CHECK(throws<std::ios_base::failure>([&] { b.saveToFileSystem(dir + "/bad", "blockmatrix"); }));
    return finish("text suite");
}

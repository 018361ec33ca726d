// The PageRank example through the compiled host mirror (include/marlin_b200.hpp): a hand-checked 4-page graph, ones for
// no iterations, and the errors.  With a path argument it also writes the ranks of the graph of
// tests/test_cpp_pagerank.py ("piece float-bits" per line) for the test to compare with the Python API bit for bit.
// Exits 3 without a GPU (there is no CPU fallback), 1 on a failed check.
#include "marlin_b200.hpp"
#include "suite.h"

#include <cstdio>
#include <cstring>

using namespace marlin;

int main(int argc, char** argv) {
    if (!require_gpu()) return 3;
    // pages 1 -> 2, 2 -> 3, 3 -> 4, 4 -> 1 (0-based rows): every rank stays 0.85 * 1 + 0.15 = 1
    SparseVecMatrix ring({{0, {1}, {1.0}}, {1, {2}, {1.0}}, {2, {3}, {1.0}}, {3, {0}, {1.0}}}, 4, 4);
    auto r = pageRank(ring, 3);
    CHECK(r.size() == 2 && r[0].size() == 2 && r[1].size() == 2);
    for (const auto& p : r)
        for (double v : p) CHECK(v == 1.0);
    // page 1 links to 2 and 3 (1/2 each), nothing else: page 2 and 3 get 0.85 * 0.5 * 1 + 0.15, pages 1 and 4 get 0.15
    SparseVecMatrix fan({{0, {1, 2}, {0.5, 0.5}}}, 5, 5);
    auto f = pageRank(fan, 1);
    CHECK(f[0].size() == 3 && f[1].size() == 2);
    CHECK(f[0][0] == 0.15 && f[0][1] == 0.85 * 0.5 + 0.15 && f[0][2] == 0.85 * 0.5 + 0.15 && f[1][0] == 0.15);
    auto ones = pageRank(fan, 0);
    CHECK(ones[0] == std::vector<double>(3, 1.0) && ones[1] == std::vector<double>(2, 1.0));

    CHECK(throws([&] { pageRank(SparseVecMatrix({{0, {1}, {1.0}}}, 3, 3), 1); }));          // one block column, two pieces
    CHECK(throws([&] { pageRank(SparseVecMatrix({{0, {1}, {1.0}}}, 4, 5), 1); }));          // not square
    CHECK(throws([&] { pageRank(SparseVecMatrix({{0, {3, 1}, {0.5, 0.5}}}, 4, 4), 1); }));  // unsorted targets

    if (argc > 1) {
        // page i (0-based) links to (7 i + 3) mod n and (i * i + 1) mod n for i not divisible by 5
        const long n = 1000;
        std::vector<SparseVecMatrix::Row> rows;
        for (long i = 0; i < n; ++i) {
            if (i % 5 == 0) continue;
            int32_t a = (int32_t)((7 * i + 3) % n), b = (int32_t)((i * i + 1) % n);
            SparseVecMatrix::Row row{i, {}, {}};
            if (a == b) { row.indices = {a}; row.values = {0.5}; }        // the same target twice: one entry of 1 / 2
            else { row.indices = {std::min(a, b), std::max(a, b)}; row.values = {0.5, 0.5}; }
            rows.push_back(row);
        }
        auto ranks = pageRank(SparseVecMatrix(rows, n, n), 12);
        std::FILE* out = std::fopen(argv[1], "w");
        for (size_t p = 0; p < ranks.size(); ++p)
            for (double v : ranks[p]) {
                uint64_t bits;
                std::memcpy(&bits, &v, 8);
                std::fprintf(out, "%zu %llu\n", p, (unsigned long long)bits);
            }
        std::fclose(out);
    }
    return finish("pagerank suite");
}

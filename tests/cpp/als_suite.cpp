// CoordinateMatrix through the compiled host mirror (include/marlin_b200.hpp): the initial factors bit for bit and two
// ALS iterations within rounding of stored expectations (tests/als_oracle.py, seed 7, rank 3, 2 x 3 blocks, lambda 0.1),
// toDenseVecMatrix with its duplicate check, the coordinate-file loader, and the argument errors.  Exits 3 without a GPU
// (there is no CPU fallback), 1 on a failed check.
#include "marlin_b200.hpp"
#include "suite.h"

#include <cmath>
#include <cstdio>
#include <fstream>
#include <unistd.h>

using namespace marlin;

int main() {
    if (!require_gpu()) return 3;
    const long r[] = {0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 0, 2, 5, 5, 1, 3};
    const long c[] = {0, 1, 1, 2, 0, 3, 2, 3, 1, 4, 4, 2, 0, 3, 4, 0};
    const float v[] = {5, 3, 4, 1, 2, 5, 3.5f, 4, 1, 2, 2.5f, 3, 4, 1.5f, 5, 2};
    std::vector<CoordinateMatrix::Entry> e;
    for (int i = 0; i < 16; ++i) e.push_back({r[i], c[i], v[i]});
    CoordinateMatrix m(e);
    CHECK(m.numRows() == 6 && m.numCols() == 5);

    // iterations = 0: the reference's initial factors (positions: users 0 2 4 | 1 3 5, products 0 3 | 1 4 | 2)
    auto init = m.ALS(3, 0, 0.1, 2, 3, false, 1.0, 7);
    CHECK((init.first.rowIds() == std::vector<long>{0, 2, 4, 1, 3, 5}));
    CHECK((init.second.rowIds() == std::vector<long>{0, 3, 1, 4, 2}));
    const DenseMatrix U0 = init.first.shard().denseBlock(), P0 = init.second.shard().denseBlock();
    CHECK(U0(0, 0) == 0.2547359041155246 && U0(0, 1) == 0.9427109305982353 && U0(0, 2) == 0.21541987021873207);
    CHECK(P0(0, 0) == 0.40789665640866629 && P0(0, 1) == 0.83231867056514419 && P0(0, 2) == 0.37532112692906272);

    // two iterations: the solve is Cholesky here, inv(A) * b in the oracle, so within rounding
    const double wantU[] = {0.26459585395995339, 1.4274754058434191, 0.27687415729025566, 1.5165108516387291, 0.026963509156918686,
                            0.65929850131826295, 0.69957885524602426, -0.2078974310826969, 0.12123430605228974, 1.2390168413926241,
                            0.51656985653610232, -0.45871003457246595, 0.89534066732016337, -0.058988206354730226, 1.258995675116199,
                            -0.14117129350714711, 1.2742624731744989, 0.12483306565152495};
    const double wantP[] = {0.89506100682115364, 3.0506951871714749, 1.0625543375174824, 2.332554303937687, 1.314111807665286,
                            1.663596118153031, 2.2587758851179953, 1.7483501443923031, -0.74392425987120969, 3.1503593879271228,
                            1.3293196303076351, -0.51711938246136879, 1.412406704206268, -0.011084679955335129, 1.5063060506928012};
    auto two = m.ALS(3, 2, 0.1, 2, 3, false, 1.0, 7);
    const DenseMatrix U = two.first.shard().denseBlock(), P = two.second.shard().denseBlock();
    double err = 0.0;
    for (int p = 0; p < 6; ++p) for (int k = 0; k < 3; ++k) err = std::max(err, std::fabs(U(p, k) - wantU[p * 3 + k]));
    for (int p = 0; p < 5; ++p) for (int k = 0; k < 3; ++k) err = std::max(err, std::fabs(P(p, k) - wantP[p * 3 + k]));
    CHECK(err <= 1e-10);
    // run to run: bit for bit
    auto again = m.ALS(3, 2, 0.1, 2, 3, false, 1.0, 7);
    CHECK(again.first.shard().denseBlock() == U && again.second.shard().denseBlock() == P);

    // toDenseVecMatrix
    CoordinateMatrix small({{0, 1, 2.5f}, {3, 0, -1.0f}, {3, 4, 7.0f}});
    DenseVecMatrix d = small.toDenseVecMatrix();
    CHECK((d.rowIds() == std::vector<long>{0, 3}));
    CHECK(d.toBreeze() == small.toBreeze());
    bool dup = false;
    try { CoordinateMatrix({{0, 1, 2.5f}, {0, 1, 1.0f}}).toDenseVecMatrix(); }
    catch (const std::invalid_argument& x) { dup = std::string(x.what()).find("Found duplicate indices: 1.") != std::string::npos; }
    CHECK(dup);

    // the loader: separators, 3 and 4 fields, and a value that must round once to float32
    char tmpl[] = "/tmp/als_suite_XXXXXX";
    const int fd = mkstemp(tmpl);
    CHECK(fd >= 0);
    close(fd);
    { std::ofstream f(tmpl); f << "1 2 3.5\n1,3,4\n2, 4, 1.00000005960464477550\n3\t5\t2.5\t881250949\n\n"; }
    CoordinateMatrix l = MTUtils::loadCoordinateMatrix(tmpl);
    std::remove(tmpl);
    CHECK(l.entries().size() == 4);
    CHECK(l.entries()[2].value == 1.0000001192092896f && (double)l.entries()[2].value == 1.0000001192092896);
    CHECK(l.entries()[3].row == 3 && l.entries()[3].col == 5 && l.entries()[3].value == 2.5f);
    CHECK(throws([] { MTUtils::loadCoordinateMatrix("relative/path"); }));

    // errors
    CHECK(throws([&] { m.ALS(129, 1, 0.1, 2, 3, false, 1.0, 7); }));
    CHECK(throws([&] { m.ALS(3, 1, -1.0, 2, 3, false, 1.0, 7); }));
    CHECK(throws([] { CoordinateMatrix({}).ALS(3, 1, 0.1, 2, 3, false, 1.0, 7); }));
    return finish("als suite");
}

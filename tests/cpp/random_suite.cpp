// The StandardNormalGenerator overloads of MTUtils in the compiled host mirror (include/marlin_b200.hpp):
// randomDenVecMatrix, randomBlockMatrix and randomSpaVecMatrix against a host restatement of the reference generator
// (java.util.Random.nextGaussian over XORShiftRandom.next, fdlibm's log), value for value.  Build with -ffp-contract=off:
// the JVM never fuses a multiply and an add.  Exits 3 without a GPU (there is no CPU fallback), 1 on a failed check.
#include "marlin_b200.hpp"
#include "suite.h"

#include <cmath>
#include <cstdio>
#include <cstring>

using namespace marlin;

// fdlibm e_log.c for positive normal x < 1
static double fdlibm_log(double x) {
    const double ln2_hi = 6.93147180369123816490e-01, ln2_lo = 1.90821492927058770002e-10;
    const double Lg1 = 6.666666666666735130e-01, Lg2 = 3.999999999940941908e-01, Lg3 = 2.857142874366239149e-01,
                 Lg4 = 2.222219843214978396e-01, Lg5 = 1.818357216161805012e-01, Lg6 = 1.531383769920937332e-01,
                 Lg7 = 1.479819860511658591e-01;
    uint64_t bits;
    std::memcpy(&bits, &x, 8);
    int32_t hx = int32_t(bits >> 32);
    int32_t k = (hx >> 20) - 1023;
    hx &= 0x000fffff;
    int32_t i = (hx + 0x95f64) & 0x100000;
    bits = (uint64_t(uint32_t(hx | (i ^ 0x3ff00000))) << 32) | (bits & 0xffffffffull);
    std::memcpy(&x, &bits, 8);
    k += i >> 20;
    const double f = x - 1.0, dk = double(k);
    if ((0x000fffff & (2 + hx)) < 3) {
        if (f == 0.0) return k == 0 ? 0.0 : dk * ln2_hi + dk * ln2_lo;
        const double R = f * f * (0.5 - 0.33333333333333333 * f);
        return k == 0 ? f - R : dk * ln2_hi - ((R - dk * ln2_lo) - f);
    }
    const double s = f / (2.0 + f), z = s * s, w = z * z;
    i = hx - 0x6147a;
    const int32_t j = 0x6b851 - hx;
    const double t1 = w * (Lg2 + w * (Lg4 + w * Lg6));
    const double t2 = z * (Lg1 + w * (Lg3 + w * (Lg5 + w * Lg7)));
    i |= j;
    const double R = t2 + t1;
    if (i > 0) {
        const double hfsq = 0.5 * f * f;
        return k == 0 ? f - (hfsq - s * (hfsq + R)) : dk * ln2_hi - ((hfsq - (s * (hfsq + R) + dk * ln2_lo)) - f);
    }
    return k == 0 ? f - s * (f - R) : dk * ln2_hi - ((s * (f - R) - dk * ln2_lo) - f);
}

// generator.copy(); setSeed(partitionSeed); nextValue() ... of StandardNormalGenerator(mean, variance)
struct Normal {
    uint64_t s;
    double mean, sd, cached = 0.0;
    bool have = false;
    Normal(int64_t partitionSeed, StandardNormalGenerator g)
        : s(uint64_t(mb_hash_seed(partitionSeed))), mean(g.mean), sd(std::sqrt(g.variance)) {}
    int64_t next(int bits) {
        s ^= s << 21;
        s ^= s >> 35;
        s ^= s << 4;
        return int64_t(s & ((1ull << bits) - 1));
    }
    double nextDouble() { return double((next(26) << 27) + next(27)) * 0x1.0p-53; }
    double nextGaussian() {
        if (have) { have = false; return cached; }
        double v1, v2, q;
        do {
            v1 = 2 * nextDouble() - 1;
            v2 = 2 * nextDouble() - 1;
            q = v1 * v1 + v2 * v2;
        } while (q >= 1 || q == 0);
        const double m = std::sqrt(-2 * fdlibm_log(q) / q);
        cached = v2 * m;
        have = true;
        return v1 * m;
    }
    double nextValue() { return mean + sd * nextGaussian(); }
};

static bool sameBits(double a, double b) { return std::memcmp(&a, &b, 8) == 0; }

int main() {
    if (!require_gpu()) return 3;
    const StandardNormalGenerator g{3.5, 0.25};

    {   // rows of 3 partitions, one stream per partition across its rows
        const long n = 37;
        const int c = 11, P = 3;
        DenseMatrix got = MTUtils::randomDenVecMatrix(n, c, P, 17, g).toBreeze();
        std::vector<int64_t> seeds(P);
        mb_partition_seeds(17, P, seeds.data());
        long start = 0, bad = 0;
        for (int p = 0; p < P; ++p) {
            const long end = (p + 1) * n / P;
            Normal ref(seeds[p], g);
            for (long r = start; r < end; ++r)
                for (int j = 0; j < c; ++j) bad += !sameBits(got(r, j), ref.nextValue());
            start = end;
        }
        CHECK(bad == 0);
    }
    {   // a 3 x 2 grid with a ragged last row and column of blocks, each block column-major
        const long n = 20, m = 15;
        DenseMatrix got = MTUtils::randomBlockMatrix(n, m, 3, 2, 18, g).toBreeze();
        const int brs = 7, bcs = 8;
        std::vector<int64_t> seeds(6);
        mb_partition_seeds(18, 6, seeds.data());
        long bad = 0;
        for (int idx = 0; idx < 6; ++idx) {
            const int bi = idx / 2, bj = idx % 2;
            const int rows = std::min<long>(brs, n - bi * brs), cols = std::min<long>(bcs, m - bj * bcs);
            Normal ref(seeds[idx], g);
            for (int cj = 0; cj < cols; ++cj)
                for (int ri = 0; ri < rows; ++ri) bad += !sameBits(got(bi * brs + ri, bj * bcs + cj), ref.nextValue());
        }
        CHECK(bad == 0);
    }
    {   // sparse rows: s values per row from the partition's normal stream, one sorted column set per partition
        const long n = 23;
        const int c = 30, P = 2, s = 6;
        SparseVecMatrix got = MTUtils::randomSpaVecMatrix(n, c, 0.2, P, 19, g);
        std::vector<int64_t> seeds(P);
        mb_partition_seeds(19, P, seeds.data());
        CHECK((long)got.rows().size() == n);
        long bad = 0;
        for (int p = 0; p < P; ++p) {
            const long start = p * n / P, end = (p + 1) * n / P;
            Normal ref(seeds[p], g);
            for (const auto& row : got.rows()) {
                if (row.id < start || row.id >= end) continue;
                CHECK((int)row.values.size() == s && row.indices == got.rows()[start].indices);
                for (int k = 1; k < (int)row.indices.size(); ++k) CHECK(row.indices[k - 1] < row.indices[k]);
            }
            for (long r = start; r < end; ++r)
                for (int k = 0; k < s; ++k) bad += !sameBits(got.rows()[r].values[k], ref.nextValue());
        }
        CHECK(bad == 0);
    }
    return finish("random suite");
}

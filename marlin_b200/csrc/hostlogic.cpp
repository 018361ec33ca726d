// Pure integer host logic of the multiply path, exported through the C ABI.
// Each function cites the reference code it mirrors (src/main/scala/edu/nju/pasalab/marlin/...).
#include "../../include/marlin_b200.h"
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

namespace {

// utils/MTUtils.scala:204-213
int dim_to_split(int64_t m, int64_t k, int64_t n) {
    if (n >= k && n >= m) return 1;
    if (m >= k && m >= n) return 2;
    return 3;
}

inline uint32_t rotl32(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }

// scala.util.hashing.MurmurHash3 (Scala 2.10 library, not in the reference tree): mix / mixLast /
// finalizeHash and bytesHash(data, arraySeed = 0x3c074a61).
uint32_t mm3_mix_last(uint32_t h, uint32_t k) {
    k *= 0xcc9e2d51u;
    k = rotl32(k, 15);
    k *= 0x1b873593u;
    return h ^ k;
}
uint32_t mm3_mix(uint32_t h, uint32_t k) {
    h = mm3_mix_last(h, k);
    h = rotl32(h, 13);
    return h * 5u + 0xe6546b64u;
}
uint32_t mm3_finalize(uint32_t h, uint32_t len) {
    h ^= len;
    h ^= h >> 16;
    h *= 0x85ebca6bu;
    h ^= h >> 13;
    h *= 0xc2b2ae35u;
    h ^= h >> 16;
    return h;
}
uint32_t mm3_bytes_hash(const uint8_t* data, int len, uint32_t seed) {
    uint32_t h = seed;
    int i = 0, rem = len;
    while (rem >= 4) {
        uint32_t k = data[i] | (uint32_t(data[i + 1]) << 8) | (uint32_t(data[i + 2]) << 16) | (uint32_t(data[i + 3]) << 24);
        h = mm3_mix(h, k);
        i += 4;
        rem -= 4;
    }
    uint32_t k = 0;
    if (rem == 3) k ^= uint32_t(data[i + 2]) << 16;
    if (rem >= 2) k ^= uint32_t(data[i + 1]) << 8;
    if (rem >= 1) {
        k ^= data[i];
        h = mm3_mix_last(h, k);
    }
    return mm3_finalize(h, uint32_t(len));
}

// java.lang.StrictMath.log (fdlibm e_log.c) for positive normal x, the only inputs nextGaussian gives it.  The C library's
// log differs from it in the last bit for some inputs (Random(42).nextGaussian() is one), and the JVM's factors are these.
double fdlibm_log(double x) {
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
    bits = (uint64_t(uint32_t(hx | (i ^ 0x3ff00000))) << 32) | (bits & 0xffffffffull);   // x or x / 2 normalised
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

// java.util.Random: the 48-bit LCG, next(bits), nextInt(), nextDouble() and nextGaussian() with its cached second value
struct JavaRandom {
    uint64_t s;
    bool have_next = false;
    double next_next = 0.0;
    explicit JavaRandom(int64_t seed) : s((uint64_t(seed) ^ 0x5DEECE66Dull) & ((1ull << 48) - 1)) {}
    int32_t next(int bits) {
        s = (s * 0x5DEECE66Dull + 0xBull) & ((1ull << 48) - 1);
        return int32_t(int64_t(s) >> (48 - bits));
    }
    double next_double() { return double((int64_t(next(26)) << 27) + next(27)) * 0x1.0p-53; }
    double next_gaussian() {
        if (have_next) {
            have_next = false;
            return next_next;
        }
        double v1, v2, q;
        do {
            v1 = 2 * next_double() - 1;
            v2 = 2 * next_double() - 1;
            q = v1 * v1 + v2 * v2;
        } while (q >= 1 || q == 0);
        const double multiplier = std::sqrt(-2 * fdlibm_log(q) / q);
        next_next = v2 * multiplier;
        have_next = true;
        return v1 * multiplier;
    }
};

// scala.util.hashing.byteswap32: v * 0x9e3775cd, Integer.reverseBytes, * 0x9e3775cd (Int arithmetic, wrapping)
int32_t byteswap32(int32_t v) {
    uint32_t hc = uint32_t(v) * 0x9e3775cdu;
    hc = (hc >> 24) | ((hc >> 8) & 0xff00u) | ((hc << 8) & 0xff0000u) | (hc << 24);
    return int32_t(hc * 0x9e3775cdu);
}

int32_t hash_block(int64_t id, int32_t n) { return int32_t(id % n); }   // HashPartitioner on a non-negative Int

}  // namespace

int32_t mb_fail(int32_t code, const char* fmt, ...);   // capi.cu: sets mb_last_error()

extern "C" {

// utils/MTUtils.scala:150-175 — CARMA-style halving of the largest dimension while cores remain.
int32_t mb_choose_split(int64_t m, int64_t k, int64_t n, int32_t cores, int32_t out_mkn[3]) {
    if (!out_mkn) return MB_ERR_INVALID_ARG;
    int ms = 1, ks = 1, ns = 1;
    int64_t _m = m, _k = k, _n = n;
    int c = cores;
    while (c > 1 && _m > 1 && _k > 1 && _n > 1) {
        const int d = dim_to_split(_m, _k, _n);
        if (d == 1) { ns *= 2; _n /= 2; }
        else if (d == 2) { ms *= 2; _m /= 2; }
        else { ks *= 2; _k /= 2; }
        c /= 2;
    }
    out_mkn[0] = ms; out_mkn[1] = ks; out_mkn[2] = ns;
    return MB_OK;
}

// matrix/DenseVecMatrix.scala:196-231 and matrix/BlockMatrix.scala:87-122.
// broadcastSize = threshold*1024*1024/8 is evaluated in Int arithmetic in the reference.
int32_t mb_choose_strategy(int64_t a_rows, int64_t a_cols, int64_t b_cols, int32_t cores,
                           int32_t broadcast_threshold_mb, int32_t other_is_block, int32_t* strategy,
                           int32_t out_mkn[3]) {
    if (!strategy || !out_mkn) return MB_ERR_INVALID_ARG;
    const int32_t broadcast_size = int32_t(uint32_t(broadcast_threshold_mb) * 1024u * 1024u) / 8;  // JVM Int wrap-around
    const int64_t b_rows = a_cols;
    out_mkn[0] = out_mkn[1] = out_mkn[2] = 0;
    if (b_rows * b_cols <= broadcast_size) { *strategy = 0; return MB_OK; }
    if (a_rows * a_cols <= broadcast_size) { *strategy = 1; return MB_OK; }
    *strategy = 2;
    if (!other_is_block) {
        // `numRows() / numCols()` is Long integer division in the reference (DenseVecMatrix.scala:210-211),
        // so the last two tests read 0.8 < floor(M/K) < 1.2, i.e. floor(M/K) == 1.
        const double ratio = double(a_rows * b_cols) / double(a_cols * a_cols);
        const int64_t q = a_cols ? a_rows / a_cols : 0;
        if (0.8 < ratio && ratio < 1.2 && double(q) < 1.2 && double(q) > 0.8) {
            const int split = int(std::floor(std::pow(3.0 * cores, 1.0 / 3.0)));
            out_mkn[0] = out_mkn[1] = out_mkn[2] = split;
            return MB_OK;
        }
    }
    return mb_choose_split(a_rows, a_cols, b_cols, cores, out_mkn);
}

// rdd/MatrixMultPartitioner.scala:12-22 with seq from matrix/BlockMatrix.scala:163,168
int32_t mb_mult_partition(int32_t i, int32_t j, int32_t kk, int32_t m, int32_t k, int32_t n) {
    (void)m;
    return i * n * k + j * k + kk;
}

// rdd/MatrixElemOpPartitioner.scala:16
int32_t mb_elem_partition(int32_t row, int32_t col, int32_t blks_by_col) { return row * blks_by_col + col; }

// matrix/BlockMatrix.scala:73-74; matrix/DenseVecMatrix.scala:1091-1094,1262-1265
int32_t mb_block_len(int64_t total, int32_t parts, int32_t* block_len, int32_t* actual_parts) {
    if (parts <= 0 || total <= 0 || !block_len || !actual_parts) return MB_ERR_INVALID_ARG;
    const int32_t len = int32_t(std::ceil(double(total) / double(parts)));
    *block_len = len;
    *actual_parts = int32_t(std::ceil(double(total) / double(len)));
    return MB_OK;
}

// utils/MTUtils.scala:18-21: ByteBuffer.allocate(java.lang.Long.SIZE /* = 64 bytes */).putLong(seed)
// -> MurmurHash3.bytesHash -> Int, widened (sign-extended) to Long.
int64_t mb_hash_seed(int64_t seed) {
    uint8_t buf[64];
    std::memset(buf, 0, sizeof(buf));
    for (int i = 0; i < 8; ++i) buf[i] = uint8_t(uint64_t(seed) >> (56 - 8 * i));   // big-endian putLong
    return int64_t(int32_t(mm3_bytes_hash(buf, 64, 0x3c074a61u)));
}

// rdd/RandomRDD.scala:28-45: partition i gets java.util.Random(seed).nextLong() (i-th draw).
int32_t mb_partition_seeds(int64_t seed, int32_t num_partitions, int64_t* seeds_out) {
    if (num_partitions < 0 || (num_partitions > 0 && !seeds_out)) return MB_ERR_INVALID_ARG;
    const uint64_t mask = (1ull << 48) - 1;
    uint64_t s = (uint64_t(seed) ^ 0x5DEECE66Dull) & mask;
    auto next32 = [&]() -> int32_t {
        s = (s * 0x5DEECE66Dull + 0xBull) & mask;
        return int32_t(s >> 16);
    };
    for (int i = 0; i < num_partitions; ++i) {
        const int64_t hi = int64_t(next32());
        const int64_t lo = int64_t(next32());
        seeds_out[i] = int64_t((uint64_t(hi) << 32) + uint64_t(lo));   // ((long)next(32) << 32) + next(32)
    }
    return MB_OK;
}

// matrix/DenseVecMatrix.scala:1565-1604 (computeSVD) and :1466-1468 (computeGramianMatrix).  The reference checks the
// column cap only where it forms the Gramian; every mode forms it here, so every mode checks it, after the mode's own
// requires.
int32_t mb_svd_mode(int64_t n, int32_t k, const char* mode, int32_t* compute_mode) {
    if (!mode || !compute_mode) return mb_fail(MB_ERR_INVALID_ARG, "mb_svd_mode: null argument");
    if (!(k > 0 && k <= n))
        return mb_fail(MB_ERR_INVALID_ARG, "Request up to n singular values but got k=%d and n=%lld.", k, (long long)n);
    int cm;
    if (std::strcmp(mode, "auto") == 0) {
        // `k > n / 2` and `k < n / 3` are Int divisions in the reference
        if (n < 100 || k > n / 2) cm = k < n / 3 ? MB_SVD_LOCAL_ARPACK : MB_SVD_LOCAL_LAPACK;
        else cm = MB_SVD_DIST_ARPACK;
    } else if (std::strcmp(mode, "local-svd") == 0) {
        cm = MB_SVD_LOCAL_LAPACK;
    } else if (std::strcmp(mode, "local-eigs") == 0) {
        cm = MB_SVD_LOCAL_ARPACK;
    } else if (std::strcmp(mode, "dist-eigs") == 0) {
        cm = MB_SVD_DIST_ARPACK;
    } else {
        return mb_fail(MB_ERR_INVALID_ARG, "Do not support mode %s.", mode);
    }
    if (cm != MB_SVD_LOCAL_LAPACK && !(k < n))
        return mb_fail(MB_ERR_INVALID_ARG, "k must be smaller than n in %s mode but got k=%d and n=%lld.",
                       cm == MB_SVD_LOCAL_ARPACK ? "local-eigs" : "dist-eigs", k, (long long)n);
    if (n > 65535) return mb_fail(MB_ERR_INVALID_ARG, "Argument with more than 65535 cols: %lld", (long long)n);
    *compute_mode = cm;
    return MB_OK;
}

// The same chooser for the overload computeSVD(k, computeU, rCond, maxIter, tol, mode) (:1557-1652), whose eigs modes
// run the Lanczos solver: the column cap belongs to computeGramianMatrix, so only the modes that form G check it.
int32_t mb_svd_plan(int64_t n, int32_t k, const char* mode, int32_t max_iter, double tol, int32_t* compute_mode) {
    (void)tol;                                         // any tol is valid: tol <= 0 asks for machine precision, as in ARPACK
    if (!mode || !compute_mode) return mb_fail(MB_ERR_INVALID_ARG, "mb_svd_plan: null argument");
    if (!(k > 0 && k <= n))
        return mb_fail(MB_ERR_INVALID_ARG, "Request up to n singular values but got k=%d and n=%lld.", k, (long long)n);
    int cm;
    if (std::strcmp(mode, "auto") == 0) {
        if (n < 100 || k > n / 2) cm = k < n / 3 ? MB_SVD_LOCAL_ARPACK : MB_SVD_LOCAL_LAPACK;
        else cm = MB_SVD_DIST_ARPACK;
    } else if (std::strcmp(mode, "local-svd") == 0) {
        cm = MB_SVD_LOCAL_LAPACK;
    } else if (std::strcmp(mode, "local-eigs") == 0) {
        cm = MB_SVD_LOCAL_ARPACK;
    } else if (std::strcmp(mode, "dist-eigs") == 0) {
        cm = MB_SVD_DIST_ARPACK;
    } else {
        return mb_fail(MB_ERR_INVALID_ARG, "Do not support mode %s.", mode);
    }
    if (cm != MB_SVD_LOCAL_LAPACK && !(k < n))
        return mb_fail(MB_ERR_INVALID_ARG, "k must be smaller than n in %s mode but got k=%d and n=%lld.",
                       cm == MB_SVD_LOCAL_ARPACK ? "local-eigs" : "dist-eigs", k, (long long)n);
    if (cm != MB_SVD_DIST_ARPACK && n > 65535)
        return mb_fail(MB_ERR_INVALID_ARG, "Argument with more than 65535 cols: %lld", (long long)n);
    if (n > INT32_MAX) return mb_fail(MB_ERR_INVALID_ARG, "Argument with more than %d cols: %lld", INT32_MAX, (long long)n);
    if (cm != MB_SVD_LOCAL_LAPACK && max_iter <= 0)
        return mb_fail(MB_ERR_INVALID_ARG, "ARPACK returns non-zero info = -4 The maximum number of Arnoldi update "
                       "iterations allowed must be greater than zero. (Refer ARPACK user guide for details)");
    *compute_mode = cm;
    return MB_OK;
}

// The projected problem of the Lanczos solver: all eigenpairs of a symmetric n x n matrix (column-major, lower triangle
// read) by cyclic Jacobi with Rutishauser's rotations, sweeping until no off-diagonal entry changes a diagonal one.
// w: eigenvalues descending (ties: lower index first); Z: the eigenvectors as columns (column-major n x n).
int32_t mb_eigs_projected(int32_t n, const double* T, double* w, double* Z) {
    if (n < 0 || (n > 0 && (!T || !w || !Z))) return mb_fail(MB_ERR_INVALID_ARG, "mb_eigs_projected: bad argument");
    std::vector<double> a((size_t)n * n), v((size_t)n * n, 0.0);
    for (int32_t j = 0; j < n; ++j)
        for (int32_t i = 0; i < n; ++i) a[(size_t)j * n + i] = i >= j ? T[(size_t)j * n + i] : T[(size_t)i * n + j];
    for (int32_t i = 0; i < n; ++i) v[(size_t)i * n + i] = 1.0;
    for (size_t i = 0; i < a.size(); ++i)
        if (!std::isfinite(a[i])) return mb_fail(MB_ERR_INVALID_ARG, "mb_eigs_projected: the matrix holds NaN or Inf");
    auto A = [&](int32_t i, int32_t j) -> double& { return a[(size_t)j * n + i]; };
    double frob = 0.0;
    for (double x : a) frob += x * x;
    // below this an entry moves no eigenvalue by more than eps^2 ||T||
    const double floor_abs = 0x1p-106 * std::sqrt(frob);
    bool rotated = true;
    for (int sweep = 0; sweep < 100 && rotated; ++sweep) {
        rotated = false;
        for (int32_t p = 0; p < n - 1; ++p)
            for (int32_t q = p + 1; q < n; ++q) {
                const double apq = A(p, q);
                if (apq == 0.0) continue;
                const double app = A(p, p), aqq = A(q, q);
                // negligible relative to both diagonal entries, or to the whole matrix
                if (std::fabs(apq) <= 0x1p-54 * std::sqrt(std::fabs(app)) * std::sqrt(std::fabs(aqq)) ||
                    std::fabs(apq) <= floor_abs) {
                    A(p, q) = A(q, p) = 0.0;
                    continue;
                }
                rotated = true;
                const double theta = (aqq - app) / (2.0 * apq);
                const double t = (theta >= 0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
                const double c = 1.0 / std::sqrt(t * t + 1.0), s = t * c, tau = s / (1.0 + c);
                for (int32_t r = 0; r < n; ++r) {
                    if (r == p || r == q) continue;
                    const double arp = A(r, p), arq = A(r, q);
                    A(r, p) = A(p, r) = arp - s * (arq + tau * arp);
                    A(r, q) = A(q, r) = arq + s * (arp - tau * arq);
                }
                A(p, p) = app - t * apq;
                A(q, q) = aqq + t * apq;
                A(p, q) = A(q, p) = 0.0;
                for (int32_t r = 0; r < n; ++r) {
                    const double vrp = v[(size_t)p * n + r], vrq = v[(size_t)q * n + r];
                    v[(size_t)p * n + r] = vrp - s * (vrq + tau * vrp);
                    v[(size_t)q * n + r] = vrq + s * (vrp - tau * vrq);
                }
            }
    }
    if (rotated) return mb_fail(MB_ERR_NO_CONVERGENCE, "mb_eigs_projected: no convergence after 100 sweeps (n = %d)", n);
    std::vector<int32_t> order(n);
    for (int32_t i = 0; i < n; ++i) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](int32_t x, int32_t y) { return A(x, x) > A(y, y); });
    for (int32_t i = 0; i < n; ++i) {
        w[i] = A(order[i], order[i]);
        std::memcpy(Z + (size_t)i * n, v.data() + (size_t)order[i] * n, sizeof(double) * n);
    }
    return MB_OK;
}

// matrix/DenseVecMatrix.scala:975-999: the reference matches "1" and "inf" (a MatchError otherwise); "fro" is its TODO,
// provided here, and "2" stays out as it does there.
int32_t mb_norm_mode(const char* mode, int32_t* kind) {
    if (!mode || !kind) return mb_fail(MB_ERR_INVALID_ARG, "mb_norm_mode: null argument");
    if (std::strcmp(mode, "1") == 0) *kind = MB_NORM_ONE;
    else if (std::strcmp(mode, "inf") == 0) *kind = MB_NORM_INF;
    else if (std::strcmp(mode, "fro") == 0) *kind = MB_NORM_FRO;
    else return mb_fail(MB_ERR_INVALID_ARG, "Do not support mode %s.", mode);
    return MB_OK;
}

// The final step of LAPACK 3.10 dnrm2 (Blue's algorithm) over accumulators added in index order.
int32_t mb_norm_fro(const double* acc, int32_t count, double* out) {
    if (!acc || !out || count <= 0) return mb_fail(MB_ERR_INVALID_ARG, "mb_norm_fro: bad argument");
    const double ssml = std::ldexp(1.0, 537), sbig = std::ldexp(1.0, -538);
    double asml = 0.0, amed = 0.0, abig = 0.0;
    for (int32_t i = 0; i < count; ++i) {
        asml += acc[3 * i];
        amed += acc[3 * i + 1];
        abig += acc[3 * i + 2];
    }
    double scl, sumsq;
    if (abig > 0.0) {
        if (amed > 0.0 || amed != amed) abig += (amed * sbig) * sbig;
        scl = 1.0 / sbig;
        sumsq = abig;
    } else if (asml > 0.0) {
        if (amed > 0.0 || amed != amed) {
            const double m = std::sqrt(amed), s = std::sqrt(asml) / ssml;
            const double ymin = s > m ? m : s, ymax = s > m ? s : m;
            scl = 1.0;
            sumsq = ymax * ymax * (1.0 + (ymin / ymax) * (ymin / ymax));
        } else {
            scl = 1.0 / ssml;
            sumsq = asml;
        }
    } else {
        scl = 1.0;
        sumsq = amed;
    }
    *out = scl * std::sqrt(sumsq);
    return MB_OK;
}

int32_t mb_sparse_check(int32_t rows, int32_t cols, const int32_t* colptr, const int32_t* rowidx) {
    if (rows < 0 || cols < 0 || !colptr) return mb_fail(MB_ERR_INVALID_ARG, "mb_sparse_check: bad argument");
    if (colptr[0] != 0) return mb_fail(MB_ERR_INVALID_ARG, "sparse block: colptr[0] is %d, not 0", colptr[0]);
    // colptr first, so that no row index past colptr[cols] (= nnz, the length of rowidx) is read
    for (int32_t j = 0; j < cols; ++j)
        if (colptr[j + 1] < colptr[j])
            return mb_fail(MB_ERR_INVALID_ARG, "sparse block: colptr decreases at column %d (%d -> %d)", j, colptr[j], colptr[j + 1]);
    if (colptr[cols] > 0 && !rowidx) return mb_fail(MB_ERR_INVALID_ARG, "mb_sparse_check: null rowidx");
    for (int32_t j = 0; j < cols; ++j) {
        const int32_t p0 = colptr[j], p1 = colptr[j + 1];
        for (int32_t p = p0; p < p1; ++p) {
            if (rowidx[p] < 0 || rowidx[p] >= rows)
                return mb_fail(MB_ERR_INVALID_ARG, "sparse block: row index %d of column %d is outside [0, %d)", rowidx[p], j, rows);
            if (p > p0 && rowidx[p] <= rowidx[p - 1])
                return mb_fail(MB_ERR_INVALID_ARG, "sparse block: row indices of column %d are not strictly increasing (%d after %d)",
                               j, rowidx[p], rowidx[p - 1]);
        }
    }
    return MB_OK;
}

// matrix/Matrices.scala:161 `(numCols * sparsity).toInt`, plus the two requires the reference lacks
int32_t mb_sparse_column_count(int32_t rows, int32_t cols, double density, int32_t* s_out) {
    if (!s_out || rows < 0 || cols < 0) return mb_fail(MB_ERR_INVALID_ARG, "mb_sparse_column_count: bad argument");
    if (!(density > 0.0))
        return mb_fail(MB_ERR_INVALID_ARG, "requirement failed: the density of sparse blocks must be positive, but got %g", density);
    const double x = (double)cols * density;
    // JVM d2i: truncate toward zero, saturate at Int.MaxValue (x > 0 here)
    const int32_t s = x >= 2147483647.0 ? INT32_MAX : (int32_t)x;
    if (s > rows)
        return mb_fail(MB_ERR_INVALID_ARG, "requirement failed: %d non-zeros per column asked of a block with %d rows "
                       "(cols * density = %d * %g)", s, rows, cols, density);
    *s_out = s;
    return MB_OK;
}

// matrix/DenseVecMatrix.scala:1607-1621
int32_t mb_svd_rank(const double* sigmas, int32_t count, int32_t k, double rcond) {
    if (count <= 0) return 0;
    if (!sigmas) return mb_fail(MB_ERR_INVALID_ARG, "mb_svd_rank: null sigmas");
    const double threshold = rcond * sigmas[0];
    int32_t i = 0;
    while (i < std::min(k, count) && sigmas[i] >= threshold) ++i;
    return i;
}

// ml/ALSHelp.scala:34-58,101-165 (ratings keyed by block with HashPartitioner, makeOutLinkBlock / makeInLinkBlock, the
// grouping and sorting of updateBlock's loop at :319-357), for the side whose ids are ent[]:
//   positions: block 0's distinct ids ascending, then block 1's, ...  (block = id mod num_blocks)
//   a position's terms: partner block ascending, partner id ascending, then input order -- i.e. the partner's position on
//   the other side ascending, ties in input order
//   work list: positions by rating count descending, ties by position
int32_t mb_als_links(int64_t nnz, const int64_t* ent, const int64_t* partner, const float* values, int32_t num_blocks,
                     int32_t num_partner_blocks, int64_t* ids_out, int64_t* block_offsets_out, int64_t* offsets_out,
                     int32_t* partners_out, float* ratings_out, int32_t* work_out, int64_t* count_out) {
    if (nnz < 0 || num_blocks < 1 || num_partner_blocks < 1 || !count_out || !block_offsets_out || !offsets_out ||
        (nnz > 0 && (!ent || !partner || !values || !ids_out || !partners_out || !ratings_out || !work_out)))
        return mb_fail(MB_ERR_INVALID_ARG, "mb_als_links: bad argument");
    if (nnz > INT32_MAX) return mb_fail(MB_ERR_UNSUPPORTED, "mb_als_links: %lld ratings (at most 2^31 - 1)", (long long)nnz);
    for (int64_t e = 0; e < nnz; ++e)
        for (int64_t id : {ent[e], partner[e]})
            if (id < 0 || id > INT32_MAX)
                return mb_fail(MB_ERR_INVALID_ARG, "ALS: id %lld of entry %lld is outside [0, 2147483647]", (long long)id,
                               (long long)e);
    // positions of both sides: distinct ids ordered by (block, id), as one monotone key (block << 31 | id)
    auto keyed = [nnz](const int64_t* ids, int32_t nb) {
        std::vector<int64_t> k((size_t)nnz);
        for (int64_t e = 0; e < nnz; ++e) k[e] = (int64_t(hash_block(ids[e], nb)) << 31) | ids[e];
        return k;
    };
    const std::vector<int64_t> ekey = keyed(ent, num_blocks), pkey = keyed(partner, num_partner_blocks);
    auto distinct = [](std::vector<int64_t> v) {
        std::sort(v.begin(), v.end());
        v.erase(std::unique(v.begin(), v.end()), v.end());
        return v;
    };
    const std::vector<int64_t> mine = distinct(ekey), theirs = distinct(pkey);
    // (entity position, partner position, input index): sorting these is the stable sort by the first two
    std::vector<std::pair<uint64_t, int32_t>> terms((size_t)nnz);
    for (int64_t e = 0; e < nnz; ++e) {
        const uint64_t ep = uint64_t(std::lower_bound(mine.begin(), mine.end(), ekey[e]) - mine.begin());
        const uint64_t pp = uint64_t(std::lower_bound(theirs.begin(), theirs.end(), pkey[e]) - theirs.begin());
        terms[e] = {(ep << 32) | pp, int32_t(e)};
    }
    std::sort(terms.begin(), terms.end());
    const int64_t n = int64_t(mine.size());
    std::fill(offsets_out, offsets_out + n + 1, 0);
    for (int64_t q = 0; q < nnz; ++q) {
        offsets_out[(terms[q].first >> 32) + 1]++;
        partners_out[q] = int32_t(terms[q].first & 0xffffffffu);
        ratings_out[q] = values[terms[q].second];
    }
    for (int64_t p = 0; p < n; ++p) offsets_out[p + 1] += offsets_out[p];
    std::fill(block_offsets_out, block_offsets_out + num_blocks + 1, 0);
    for (int64_t p = 0; p < n; ++p) {
        ids_out[p] = mine[p] & INT32_MAX;
        block_offsets_out[(mine[p] >> 31) + 1]++;
        work_out[p] = int32_t(p);
    }
    for (int32_t b = 0; b < num_blocks; ++b) block_offsets_out[b + 1] += block_offsets_out[b];
    std::stable_sort(work_out, work_out + n, [&](int32_t a, int32_t b) {
        return offsets_out[a + 1] - offsets_out[a] > offsets_out[b + 1] - offsets_out[b];
    });
    *count_out = n;
    return MB_OK;
}

// ml/ALSHelp.scala:60-74,170-179: seed1 / seed2 are the first two nextInt() of Random(seed); block b of the users (side 0)
// or products (side 1) draws from Random(byteswap32(seed1 or seed2 ^ b)), and its p-th position gets the p-th
// randomFactor: rank draws of |nextGaussian()| over the square root of their in-order sum of squares.
int32_t mb_als_init_factors(int64_t seed, int32_t side, int32_t block, int32_t rank, int64_t count, double* out) {
    if ((side != 0 && side != 1) || block < 0 || rank < 1 || count < 0 || (count > 0 && !out))
        return mb_fail(MB_ERR_INVALID_ARG, "mb_als_init_factors: bad argument");
    JavaRandom gen(seed);
    const int32_t seed1 = gen.next(32), seed2 = gen.next(32);
    JavaRandom rand(int64_t(byteswap32((side == 0 ? seed1 : seed2) ^ block)));
    for (int64_t p = 0; p < count; ++p) {
        double* f = out + p * rank;
        double sum = 0.0;
        for (int32_t i = 0; i < rank; ++i) f[i] = std::fabs(rand.next_gaussian());
        for (int32_t i = 0; i < rank; ++i) sum += f[i] * f[i];
        const double norm = std::sqrt(sum);
        for (int32_t i = 0; i < rank; ++i) f[i] = f[i] / norm;
    }
    return MB_OK;
}

// examples/PageRank.scala:13-27 (the link rows) and DenseVecMatrix.scala:1420-1436 (their transpose): the in-link rows of
// targets [t0, t1), sources ascending.  A stable counting sort by target over the link rows taken in ascending source id:
// count, scan, place.
int32_t mb_pagerank_links(int32_t n, int64_t num_rows, const int64_t* ids, const int64_t* rowptr, const int32_t* targets,
                          const double* values, int32_t t0, int32_t t1, double damping, int32_t* in_rowptr_out,
                          int32_t* sources_out, double* weights_out, int64_t* nnz_out) {
    if (n < 0 || num_rows < 0 || !rowptr || !in_rowptr_out || !nnz_out || (num_rows > 0 && !ids))
        return mb_fail(MB_ERR_INVALID_ARG, "mb_pagerank_links: bad argument");
    if (t0 < 0 || t1 < t0 || t1 > n)
        return mb_fail(MB_ERR_INVALID_ARG, "PageRank: target range [%d, %d) is outside [0, %d]", t0, t1, n);
    if (rowptr[0] != 0) return mb_fail(MB_ERR_INVALID_ARG, "PageRank: rowptr[0] is %lld, not 0", (long long)rowptr[0]);
    std::vector<int64_t> order((size_t)num_rows);
    for (int64_t r = 0; r < num_rows; ++r) {
        if (ids[r] < 0 || ids[r] >= n)
            return mb_fail(MB_ERR_INVALID_ARG, "PageRank: source page %lld is outside [0, %d)", (long long)ids[r], n);
        if (rowptr[r + 1] < rowptr[r])
            return mb_fail(MB_ERR_INVALID_ARG, "PageRank: rowptr decreases at row %lld", (long long)r);
        if (rowptr[r + 1] > rowptr[r] && (!targets || !values))
            return mb_fail(MB_ERR_INVALID_ARG, "mb_pagerank_links: null targets or values");
        for (int64_t q = rowptr[r]; q < rowptr[r + 1]; ++q) {
            if (targets[q] < 0 || targets[q] >= n)
                return mb_fail(MB_ERR_INVALID_ARG, "PageRank: target page %d of source page %lld is outside [0, %d)",
                               targets[q], (long long)ids[r], n);
            if (q > rowptr[r] && targets[q] <= targets[q - 1])
                return mb_fail(MB_ERR_INVALID_ARG, "PageRank: the targets of source page %lld are not strictly increasing",
                               (long long)ids[r]);
        }
        order[r] = r;
    }
    std::sort(order.begin(), order.end(), [ids](int64_t a, int64_t b) { return ids[a] < ids[b]; });
    for (int64_t r = 1; r < num_rows; ++r)
        if (ids[order[r]] == ids[order[r - 1]])
            return mb_fail(MB_ERR_INVALID_ARG, "PageRank: source page %lld has two link rows", (long long)ids[order[r]]);
    const int32_t m = t1 - t0;
    std::vector<int64_t> count((size_t)m + 1, 0);
    for (int64_t q = 0; q < (num_rows ? rowptr[num_rows] : 0); ++q)
        if (targets[q] >= t0 && targets[q] < t1) ++count[targets[q] - t0 + 1];
    for (int32_t k = 0; k < m; ++k) count[k + 1] += count[k];
    if (count[m] > INT32_MAX)
        return mb_fail(MB_ERR_UNSUPPORTED, "PageRank: %lld in-links in one range, at most 2^31 - 1", (long long)count[m]);
    if (count[m] > 0 && (!sources_out || !weights_out)) return mb_fail(MB_ERR_INVALID_ARG, "mb_pagerank_links: null output");
    for (int32_t k = 0; k <= m; ++k) in_rowptr_out[k] = (int32_t)count[k];
    for (int64_t r : order)
        for (int64_t q = rowptr[r]; q < rowptr[r + 1]; ++q) {
            const int32_t t = targets[q];
            if (t < t0 || t >= t1) continue;
            const int64_t at = count[t - t0]++;
            sources_out[at] = (int32_t)ids[r];
            weights_out[at] = values[q] * damping;
        }
    *nnz_out = in_rowptr_out[m];
    return MB_OK;
}

}  // extern "C"

"""The fp64 kernels away from unit scale, on IEEE special values, on exact ties and on views inside poisoned parents.

Every bitwise assertion here rests on one of three facts, stated next to it:
  * power-of-two scaling is exact: multiplying every input by 2^k multiplies every product, sum, quotient and square
    root the kernels form by a fixed power of two, without changing a bit of any significand, as long as no
    intermediate leaves the normal range (|x| in [2^-1022, 2^1024)).  So a kernel must reproduce its own unscaled
    result, scaled, bit for bit, whatever its summation order, tiling or split;
  * integer (or dyadic) data whose every partial sum fits in 53 bits is computed without rounding in any order;
  * a transpose or a view is a copy: nothing is computed.
Tolerances are stated where a result is compared with a rounded reference.
"""
import ctypes as C
import math

import numpy as np
import pytest

from marlin_b200 import _native as nat
from tests import exact_oracle as eo
from tests.harness import gpu  # noqa: F401  (a fixture)
from tests.test_gpu_cabi import alloc, download, upload_mat

pytestmark = pytest.mark.gpu
EPS = np.finfo(np.float64).eps


# ------------------------------------------------------------------------------------------------------------ helpers
def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def identical(a, b):
    """Bit for bit, -0.0 != 0.0 and NaN payloads included."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and np.array_equal(bits(a), bits(b))


def same(a, b):
    """Bitwise, except that any NaN equals any NaN (device and host may pick different payloads)."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    if a.shape != b.shape or not np.array_equal(np.isnan(a), np.isnan(b)):
        return False
    keep = ~np.isnan(a)
    return np.array_equal(bits(a[keep]), bits(b[keep]))


def equal_values(a, b):
    """Equal as numbers (-0.0 == 0.0), shapes included.  For exact integer / dyadic work: every value is exact in any
    order, but the sign of a zero result is not a matter of rounding — 0 * (1 / pivot) is -0.0 for a negative pivot, and
    x - x is +0.0 while fma(-l, u, a) may give -0.0 — so it may differ between summation orders."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and np.array_equal(a, b)


def p2(k):
    return math.ldexp(1.0, int(k))


def cuda(x):
    """A flat column-major float64 torch tensor on the GPU holding the 2-D array x (or a flat array as is)."""
    import torch
    x = np.asarray(x, dtype=np.float64)
    flat = x.reshape(-1, order="F") if x.ndim == 2 else x
    t = torch.from_numpy(np.ascontiguousarray(flat)).cuda()
    torch.cuda.synchronize()
    return t


def ptr(t):
    return C.c_void_p(t.data_ptr())


def colmajor_host(t, rows, cols, ld, offset=0):
    h = t.cpu().numpy()
    return np.array([h[offset + j * ld: offset + j * ld + rows] for j in range(cols)]).T.reshape(rows, cols)


def wrap(gpu, t, rows, cols, ld, offset=0, trans=0):
    lib, ctx = gpu
    h = nat.c_blk()
    nat.check(lib.mb_block_wrap(ctx, ptr(t), offset, rows, cols, ld, trans, nat.MB_F64, C.byref(h)))
    return h


def sync(gpu):
    nat.check(gpu[0].mb_synchronize(gpu[1]))


def dgemm(gpu, A, B, ta=0, tb=0, C0=None, beta=0.0, alpha=1.0, generic=False):
    """C = alpha op(A) op(B) + beta C0 through mb_dgemm_device (or the CUDA-core kernel); A, B are the logical
    operands; op(X) = X with X^T stored when the flag is set.  C0 = None: C starts as NaN (beta = 0 must not read it)."""
    lib, ctx = gpu
    m, k = A.shape
    n = B.shape[1]
    dA, dB = cuda(A.T if ta else A), cuda(B.T if tb else B)
    dC = cuda(np.full((m, n), np.nan) if C0 is None else C0)
    fn = lib.mb_dgemm_device_generic if generic else lib.mb_dgemm_device
    nat.check(fn(ctx, b"T" if ta else b"N", b"T" if tb else b"N", m, n, k, alpha, ptr(dA), max(1, k if ta else m), ptr(dB),
                 max(1, n if tb else k), beta, ptr(dC), max(1, m)))
    sync(gpu)
    return colmajor_host(dC, m, n, max(1, m))


def split_gemm(gpu, A, B, C0=None, slices=7, mode=1):
    lib, ctx = gpu
    nat.check(lib.mb_set_fp64_mode(ctx, mode, slices))
    try:
        return dgemm(gpu, A, B, C0=C0, beta=0.0 if C0 is None else 1.0)
    finally:
        nat.check(lib.mb_set_fp64_mode(ctx, 0, 7))


def away_from_zero(rng, shape, lo=0.5):
    """Random signs times U[lo, 1): no entry is tiny, so scaling by 2^-k keeps every input normal."""
    return np.where(rng.random(shape) < 0.5, -1.0, 1.0) * (lo + (1 - lo) * rng.random(shape))


# =============================================================================== B. power-of-two scaling, bit for bit
# Standard-normal operands lie in [2^-20, 2^3] here; a product of two is >= 2^-40, and any partial sum of K <= 400
# such products that does not cancel to zero is a multiple of ulp(2^-40) = 2^-92.  So with a combined scale 2^s,
# |s| <= 900, every intermediate stays within [2^-992, 2^920]: normal.
GEMM_SCALES = [(300, 300), (-300, -300), (500, -500), (-500, 400), (500, 400), (-500, -400)]


@pytest.mark.parametrize("generic", [False, True])
@pytest.mark.parametrize("ta", [0, 1])
@pytest.mark.parametrize("tb", [0, 1])
def test_gemm_power_of_two_scaling(gpu, ta, tb, generic):
    m, n, k = 300, 260, 333                    # ragged against the 128-wide tiles, several tiles each way
    rng = np.random.default_rng(10 * ta + tb + 100 * generic)
    A, B = rng.standard_normal((m, k)), rng.standard_normal((k, n))
    C0 = rng.standard_normal((m, n))
    base = dgemm(gpu, A, B, ta, tb, generic=generic)
    base_acc = dgemm(gpu, A, B, ta, tb, C0=C0, beta=1.0, generic=generic)
    for ea, eb in GEMM_SCALES[:3] if generic else GEMM_SCALES:
        s = p2(ea + eb)
        assert identical(dgemm(gpu, A * p2(ea), B * p2(eb), ta, tb, generic=generic), base * s), (ea, eb)
        assert identical(dgemm(gpu, A * p2(ea), B * p2(eb), ta, tb, C0=C0 * s, beta=1.0, generic=generic), base_acc * s)
    # per-row scaling of A and per-column scaling of B: (D_r A)(B D_c) = D_r (A B) D_c, exponents within +-400 so
    # |r_i + c_j| <= 800 (same range argument as above)
    r = rng.integers(-400, 401, size=m).astype(float)
    c = rng.integers(-400, 401, size=n).astype(float)
    Dr, Dc = np.exp2(r), np.exp2(c)
    got = dgemm(gpu, Dr[:, None] * A, B * Dc[None, :], ta, tb, generic=generic)
    assert identical(got, Dr[:, None] * base * Dc[None, :])


def test_int8_split_power_of_two_scaling(gpu):
    """The split keeps one exponent per row of A (eA) and per column of B (eB); rescaling rows and columns by 2^r_i, 2^c_j
    with |r_i|, |c_j| <= 450 must move only those exponents: every digit, every int32 sum and every fold term is the
    same, scaled.  Inputs in [0.5, 1) in magnitude: the smallest fold weight is 2^(eA+eB-2P+7(s-1)) >= 2^-958, normal."""
    m, n, k = 384, 320, 512
    rng = np.random.default_rng(21)
    A, B = away_from_zero(rng, (m, k)), away_from_zero(rng, (k, n))
    C0 = rng.standard_normal((m, n))
    base = split_gemm(gpu, A, B)
    base_acc = split_gemm(gpu, A, B, C0=C0)
    r = rng.integers(-450, 451, size=m).astype(float)
    c = rng.integers(-450, 451, size=n).astype(float)
    r[:5], c[:5] = 450, -450
    Dr, Dc = np.exp2(r), np.exp2(c)
    S = Dr[:, None] * Dc[None, :]
    assert identical(split_gemm(gpu, Dr[:, None] * A, B * Dc[None, :]), base * S)
    assert identical(split_gemm(gpu, Dr[:, None] * A, B * Dc[None, :], C0=C0 * S), base_acc * S)
    for ea, eb in [(450, 400), (-450, -400), (450, -450)]:
        assert identical(split_gemm(gpu, A * p2(ea), B * p2(eb)), base * p2(ea + eb))
    # the same through the Python runtime's mode switch and the block API
    import marlin_b200 as mb
    rt = mb.Runtime.get()
    rt.set_fp64_mode("int8x7", 7)
    try:
        got0 = mb.SubMatrix(A).multiply(mb.SubMatrix(B)).toBreeze()
        got1 = mb.SubMatrix(Dr[:, None] * A).multiply(mb.SubMatrix(B * Dc[None, :])).toBreeze()
    finally:
        rt.set_fp64_mode("native")
    assert identical(got0, base) and identical(got1, base * S)


def test_bf16_gemm_power_of_two_scaling(gpu):
    """bf16 operands, fp32 result.  bf16 and fp32 share the exponent range 2^-126..2^127; inputs of magnitude [0.5, 1)
    (exact in bf16 after rounding, which commutes with 2^k) and scales (a, b) with |a + b| <= 80 keep products within
    2^-82..2^90 and every fp32 partial sum's ulp above 2^-110: normal."""
    lib, ctx = gpu
    m, n, k = 200, 264, 256
    rng = np.random.default_rng(31)
    A, B = away_from_zero(rng, (m, k)), away_from_zero(rng, (k, n))

    def run(X, Y):
        ha, hb = upload_mat(gpu, X, nat.MB_BF16), upload_mat(gpu, Y, nat.MB_BF16)
        hc = alloc(gpu, m, n, nat.MB_F32)
        nat.check(lib.mb_block_gemm(ctx, ha, hb, hc, 0))
        return download(gpu, hc, m, n)
    base = run(A, B)
    for ea, eb in [(60, -60), (-60, 60), (40, 40), (-40, -40)]:
        assert identical(run(A * p2(ea), B * p2(eb)), base * p2(ea + eb)), (ea, eb)


def test_gemv_dot_ger_power_of_two_scaling(gpu):
    """Scales (a, b) with |a + b| <= 900 on standard-normal data: the range argument of the GEMM above."""
    lib, ctx = gpu
    m, n = 1000, 700                          # two column chunks of the N kernel, several row segments of the T kernel
    rng = np.random.default_rng(41)
    A, x, xt = rng.standard_normal((m, n)), rng.standard_normal(n), rng.standard_normal(m)

    def gemv(M, x, trans=False):
        """y = M x; trans: M is a transposed view (M^T stored), which runs the T kernel."""
        ha = upload_mat(gpu, M.T if trans else M)
        if trans:
            v = nat.c_blk()
            nat.check(lib.mb_block_view_t(ctx, ha, C.byref(v)))
            ha = v
        rows = M.shape[0]
        hx, hy = upload_mat(gpu, x[:, None]), alloc(gpu, rows, 1)
        nat.check(lib.mb_block_gemv(ctx, ha, hx, hy, 0))
        return download(gpu, hy, rows, 1)[:, 0]

    def dot(x, y):
        out = C.c_double()
        nat.check(lib.mb_block_dot(ctx, upload_mat(gpu, x[:, None]), upload_mat(gpu, y[:, None]), C.byref(out)))
        return out.value

    def ger(x, y):
        ho = alloc(gpu, len(x), len(y))
        nat.check(lib.mb_block_ger(ctx, upload_mat(gpu, x[:, None]), upload_mat(gpu, y[None, :]), ho))
        return download(gpu, ho, len(x), len(y))
    base_n, base_t = gemv(A, x), gemv(A.T, xt, trans=True)
    base_d, base_g = dot(x, A[0, :]), ger(xt[:300], x[:200])
    for ea, eb in [(500, 400), (-500, -400), (450, -450)]:
        s = p2(ea + eb)
        assert identical(gemv(A * p2(ea), x * p2(eb)), base_n * s)
        assert identical(gemv(A.T * p2(ea), xt * p2(eb), trans=True), base_t * s)
        assert identical(np.float64(dot(x * p2(ea), A[0, :] * p2(eb))), np.float64(base_d * s))
        assert identical(ger(xt[:300] * p2(ea), x[:200] * p2(eb)), base_g * s)


def _rowshard(A):
    import torch
    import marlin_b200 as mb
    m, n = A.shape
    buf = torch.from_numpy(np.ascontiguousarray(A).reshape(-1)).cuda()
    return mb.SubMatrix(buf=buf, rows=m, cols=n, ld=max(1, n), is_transpose=True)


@pytest.mark.parametrize("n", [2816, 3000])             # split-K (fewer than two waves of triangle tiles) and unsplit
def test_gramian_power_of_two_scaling(n):
    """A 2^k -> 4^k G with |k| <= 200, and A D -> D G D with D's exponents within +-150: entries of A in [2^-20, 2^3],
    products >= 2^-40, partial sums multiples of >= 2^-92 (m = 64), so everything stays within [2^-492, 2^410]."""
    import marlin_b200 as mb
    m = 64
    rng = np.random.default_rng(n)
    A = rng.standard_normal((m, n))
    d = np.exp2(rng.integers(-150, 151, size=n).astype(float))
    for make in (_rowshard, mb.SubMatrix):
        G = make(A).gramian().toBreeze()
        for k in (200, -200):
            assert identical(make(A * p2(k)).gramian().toBreeze(), G * p2(2 * k)), (make, k)
        assert identical(make(A * d[None, :]).gramian().toBreeze(), d[:, None] * G * d[None, :]), make


def lu_gpu(gpu, A):
    lib, ctx = gpu
    h = upload_mat(gpu, A)
    perm = (C.c_int32 * A.shape[0])()
    nat.check(lib.mb_block_lu(ctx, h, perm))
    return download(gpu, h, *A.shape), np.array(perm[:], dtype=np.int64)


@pytest.mark.parametrize("n", [200, 257])
def test_lu_power_of_two_scaling(gpu, n):
    """Partial pivoting compares entries of one column, all scaled alike, so A 2^k and A D pivot exactly as A does; L is
    a ratio of entries of one column (unchanged) and U takes the column's scale.  Entries of A in [2^-20, 1], growth of
    U small for random data: with |k| and D's exponents <= 300 everything stays normal."""
    rng = np.random.default_rng(n + 7)
    A = rng.random((n, n)) - 0.5
    base, perm = lu_gpu(gpu, A)
    L, U = np.tril(base, -1), np.triu(base)
    for k in (300, -300):
        got, p = lu_gpu(gpu, A * p2(k))
        assert np.array_equal(p, perm) and identical(got, L + U * p2(k)), k
    d = np.exp2(rng.integers(-300, 301, size=n).astype(float))
    got, p = lu_gpu(gpu, A * d[None, :])
    assert np.array_equal(p, perm) and identical(got, L + U * d[None, :])


def cholesky_gpu(gpu, A):
    lib, ctx = gpu
    h = upload_mat(gpu, A)
    nat.check(lib.mb_block_cholesky(ctx, h))
    return download(gpu, h, *A.shape)


def test_cholesky_power_of_two_scaling(gpu):
    """4^k A = (2^k L)(2^k L)^T and D A D = (D L)(D L)^T: square roots of 4^k x and quotients by 2^k y are exact."""
    n = 200
    rng = np.random.default_rng(51)
    G = rng.standard_normal((n, n))
    A = G @ G.T + n * np.eye(n)
    L = cholesky_gpu(gpu, A)
    for k in (200, -200):
        assert identical(cholesky_gpu(gpu, A * p2(2 * k)), L * p2(k)), k
    d = np.exp2(rng.integers(-200, 201, size=n).astype(float))
    assert identical(cholesky_gpu(gpu, d[:, None] * A * d[None, :]), d[:, None] * L)


def test_trsm_and_inverse_power_of_two_scaling(gpu):
    """(2^a T) X' = 2^b B gives X' = 2^(b-a) X; (2^k A)^-1 = 2^-k A^-1.  Exponents <= 300: entries stay normal."""
    lib, ctx = gpu
    rng = np.random.default_rng(61)
    t, nrhs = 300, 70
    T = np.tril(rng.random((t, t)) - 0.5) + 4 * np.eye(t)
    B = rng.random((t, nrhs)) - 0.5

    def trsm(T, B):
        hb = upload_mat(gpu, B)
        nat.check(lib.mb_block_trsm(ctx, upload_mat(gpu, T), 1, 0, hb))
        return download(gpu, hb, *B.shape)

    def inv(A):
        ho = alloc(gpu, *A.shape)
        nat.check(lib.mb_block_inverse(ctx, upload_mat(gpu, A), ho))
        return download(gpu, ho, *A.shape)
    X = trsm(T, B)
    for a, b in [(300, -200), (-300, 250)]:
        assert identical(trsm(T * p2(a), B * p2(b)), X * p2(b - a)), (a, b)
    A = rng.random((257, 257)) - 0.5 + 2 * np.eye(257)
    Ai = inv(A)
    for k in (300, -300):
        assert identical(inv(A * p2(k)), Ai * p2(-k)), k


def _sym_test_matrix(n, seed, definite):
    """A symmetric matrix with entries of magnitude >= 2^-12 (so 2^-1000 G keeps every entry normal) and eigenvalues of
    magnitude >= 2^-12 (so 2^-1000 w stays normal)."""
    rng = np.random.default_rng(seed)
    S = away_from_zero(rng, (n, n), lo=2.0 ** -12)
    G = S @ S.T / n + 0.25 * np.eye(n) if definite else (S + S.T) / 2
    G[np.abs(G) < 2.0 ** -12] = 2.0 ** -12
    G = np.tril(G) + np.tril(G, -1).T
    w = np.linalg.eigvalsh(G)
    assert np.abs(w).min() >= 2.0 ** -12
    return G


@pytest.mark.parametrize("definite", [True, False])
def test_jacobi_power_of_two_scaling(definite):
    """symmetricEigen of 2^k G: V and the sweep count identical to G's, w scaled by 2^k exactly.  With k = +-520 and
    beyond, g_pp g_qq used to overflow (or underflow), so the solver skipped every rotation (or never stopped)."""
    import marlin_b200 as mb
    n = 40
    G = _sym_test_matrix(n, 71 + definite, definite)
    blk = mb.SubMatrix(G)
    w, V = blk.symmetricEigen()
    V, sweeps = V.toBreeze(), blk.last_sweeps
    assert np.abs(w - sorted(np.linalg.eigvalsh(G), key=lambda x: -abs(x))).max() <= 1e-12 * np.abs(w).max()
    for k in (520, -520, 900, -900, -1000):
        b = mb.SubMatrix(G * p2(k))
        wk, Vk = b.symmetricEigen()
        assert identical(Vk.toBreeze(), V) and b.last_sweeps == sweeps, k
        assert identical(wk, w * p2(k)), k


def test_jacobi_2x2_at_2_to_531():
    """2^531 [[2, 1], [1, 2]]: one rotation with t = 1 gives the eigenvalues 3 and 1 exactly (times 2^531)."""
    import marlin_b200 as mb
    w, _ = mb.SubMatrix(np.array([[2.0, 1.0], [1.0, 2.0]]) * p2(531)).symmetricEigen()
    assert identical(w, np.array([3.0, 1.0]) * p2(531))


def test_compute_svd_power_of_two_scaling():
    """computeSVD of 2^k A: G = 4^k A^T A, s = sqrt(4^k w) = 2^k s, V identical, U = (2^k A) V (2^-k S^-1) identical.
    Entries of A in [2^-20, 2^3], m = 300: every intermediate stays normal for k in {-400, 260, 400}."""
    import marlin_b200 as mb
    rng = np.random.default_rng(81)
    A = rng.standard_normal((300, 40))
    U, s, V = mb.DenseVecMatrix(list(enumerate(A))).computeSVD(10, computeU=True)
    U = U.toBreeze()
    for k in (-400, 260, 400):
        Uk, sk, Vk = mb.DenseVecMatrix(list(enumerate(A * p2(k)))).computeSVD(10, computeU=True)
        assert identical(Vk, V) and identical(sk, s * p2(k)) and identical(Uk.toBreeze(), U), k


# ========================================================================================== C. IEEE special values
SPECIALS = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, 5e-324, -5e-324, 2.2250738585072014e-308, 1.7976931348623157e308,
                     -1.7976931348623157e308, 1.0, -3.5, 1e-310, 2.0 ** 1023, 0.1])


def _special_pair(rng, m, n):
    a = rng.choice(SPECIALS, size=(m, n))
    b = rng.choice(SPECIALS, size=(m, n))
    a[: len(SPECIALS), 0] = SPECIALS                 # every special against every special in the first columns
    b[: len(SPECIALS), :len(SPECIALS)] = SPECIALS[None, :]
    a[: len(SPECIALS), :len(SPECIALS)] = SPECIALS[:, None]
    return a, b


def test_elementwise_special_values_bit_exact(gpu):
    """add, sub, hadamard, axpb and div are single IEEE operations (two for axpb, rounded separately): bit-exact against
    numpy, NaN payloads aside."""
    lib, ctx = gpu
    m, n = 40, 33
    A, B = _special_pair(np.random.default_rng(91), m, n)
    ha, hb = upload_mat(gpu, A), upload_mat(gpu, B)

    def run2(fn):
        ho = alloc(gpu, m, n)
        nat.check(fn(ctx, ha, hb, ho))
        return download(gpu, ho, m, n)
    with np.errstate(all="ignore"):
        assert same(run2(lib.mb_block_add), A + B)
        assert same(run2(lib.mb_block_sub), A - B)
        assert same(run2(lib.mb_block_hadamard), A * B)
        for alpha, beta in [(2.0, -0.5), (-1.0, np.inf), (0.0, 1.0), (1e308, -1e308)]:
            ho = alloc(gpu, m, n)
            nat.check(lib.mb_block_axpb(ctx, ha, alpha, beta, ho))
            assert same(download(gpu, ho, m, n), alpha * A + beta), (alpha, beta)
        for b in (0.0, -0.0, 3.0, np.inf, -np.inf, np.nan, 5e-324):
            for b_over_a in (0, 1):
                ho = alloc(gpu, m, n)
                nat.check(lib.mb_block_div(ctx, ha, b, b_over_a, ho))
                want = b / A if b_over_a else A / b
                assert same(download(gpu, ho, m, n), want), (b, b_over_a)


def test_transpose_copies_bits(gpu):
    """A transpose is a copy: -0.0 and NaN payloads (quiet, negative, with payload bits) survive."""
    lib, ctx = gpu
    m, n = 70, 45
    A, _ = _special_pair(np.random.default_rng(92), m, n)
    raw = bits(A).copy()
    raw[3, 4] = 0x7FF8000000001234
    raw[5, 6] = np.int64(-0x0007FFFFFFFFABCD)          # 0xFFF8...5433: a negative quiet NaN with a payload
    A = raw.view(np.float64)
    ho = alloc(gpu, n, m)
    nat.check(lib.mb_block_transpose(ctx, upload_mat(gpu, A), ho))
    assert identical(download(gpu, ho, n, m), A.T)


def test_sum_special_values(gpu):
    """sum gives NaN or +-Inf as IEEE does: any NaN or both infinities -> NaN, one sign of infinity -> that infinity."""
    lib, ctx = gpu
    rng = np.random.default_rng(93)
    for extra, want in [([np.inf], np.inf), ([-np.inf], -np.inf), ([np.inf, -np.inf], np.nan), ([np.nan], np.nan),
                        ([np.inf, np.nan], np.nan)]:
        A = rng.standard_normal((300, 70))
        idx = rng.choice(A.size, size=len(extra), replace=False)
        A.reshape(-1)[idx] = extra
        out = C.c_double()
        nat.check(lib.mb_block_sum(ctx, upload_mat(gpu, A), C.byref(out)))
        assert same(np.float64(out.value), np.float64(want)), extra


def bf16_rne(x):
    """fp64 -> bf16 (as the fp64 value it stands for) by round-to-nearest-even in integer arithmetic on the fp64
    significand: 8 significant bits, fp32's exponent range (normal down to 2^-126, subnormal steps of 2^-133), overflow
    to +-Inf, zeros and NaN kept."""
    out = np.empty(x.shape)
    for i, v in enumerate(x):
        if math.isnan(v) or math.isinf(v) or v == 0.0:
            out[i] = v
            continue
        fm, fe = math.frexp(abs(v))                # |v| = fm 2^fe, fm in [0.5, 1)
        sig = int(fm * 2 ** 53)                    # |v| = sig 2^(fe - 53), exactly
        q = max(fe - 8, -133)                      # the bf16 quantum at |v|
        shift = q - (fe - 53)                      # > 0: fp64 has 53 significant bits, bf16 8
        r, rem = divmod(sig, 1 << shift)
        half = 1 << (shift - 1)
        if rem > half or (rem == half and r & 1):
            r += 1
        val = math.inf if q + r.bit_length() > 128 else math.ldexp(r, q)       # >= 2^128: beyond bf16's range
        out[i] = math.copysign(val, v)
    return out


def test_bf16_upload_rounds_to_nearest_even(gpu):
    """Exact ties (both parities), values just above and below a tie, overflow to +-Inf (and the largest value that still
    rounds down to bf16 max), bf16 subnormals and their ties, -0.0, NaN."""
    lib, ctx = gpu
    ulp1 = 2.0 ** -7                                 # bf16 spacing in [1, 2)
    vals = [1 + ulp1 / 2, 1 + 3 * ulp1 / 2, 1 + ulp1 / 2 + 2.0 ** -40, 1 + ulp1 / 2 - 2.0 ** -40, -(1 + ulp1 / 2),
            3.3895313892515355e38, 3.3895313892515355e38 * (1 + 2.0 ** -9), 3.3895313892515355e38 * (1 + 2.0 ** -8.5),
            1e39, -1e39, 1.7976931348623157e308, 2.0 ** -126, 2.0 ** -130, 2.0 ** -133, 2.0 ** -134, 3 * 2.0 ** -134,
            2.0 ** -134 * 1.0000001, 2.0 ** -135, 2.0 ** -140, 5e-324, -0.0, 0.0, np.nan, -np.inf, np.inf, 0.1, -1e-40,
            np.pi * 2.0 ** 100]
    x = np.array(vals)
    h = upload_mat(gpu, x[:, None], nat.MB_BF16)
    got = download(gpu, h, len(x), 1)[:, 0]
    assert same(got, bf16_rne(x)), np.flatnonzero(~np.isclose(got, bf16_rne(x), equal_nan=True))


def test_gemv_skips_zero_x_like_f2j(gpu, oracle):
    """dgemv 'N' skips column j when x(j) = 0, so an Inf or NaN in that column never reaches y: bit-identical to the
    F2J restatement (one column chunk: the same summation order), in the vector and the scalar path."""
    lib, ctx = gpu
    rng = np.random.default_rng(101)
    for m in (300, 301):                              # even rows: double2 loads; odd: the scalar tail row
        n = 200
        A, x = rng.standard_normal((m, n)), rng.standard_normal(n)
        x[[3, 17, 18, 150]] = 0.0
        x[19] = -0.0
        A[:, 3] = np.inf
        A[5, 17] = np.nan
        A[::3, 18] = -np.inf
        A[7, 19] = np.nan
        A[9, 20] = np.inf                              # x(20) != 0: this one propagates
        ha, hx, hy = upload_mat(gpu, A), upload_mat(gpu, x[:, None]), alloc(gpu, m, 1)
        nat.check(lib.mb_block_gemv(ctx, ha, hx, hy, 0))
        got = download(gpu, hy, m, 1)[:, 0]
        want = oracle.block_multiply_vector(np.asfortranarray(A), x)
        assert same(got, want), m
        assert np.isfinite(got[np.arange(m) != 9]).all()


def _explicit_product(A, B):
    """IEEE sum of the elementwise products, no zero skipped: the class (finite / NaN / +Inf / -Inf) of each entry does
    not depend on the summation order (the finite entries here stay far from overflow)."""
    with np.errstate(all="ignore"):
        return (A[:, :, None] * B[None, :, :]).sum(1)


def _classes(X):
    return np.where(np.isnan(X), 3, np.where(X == np.inf, 1, np.where(X == -np.inf, 2, 0)))


@pytest.mark.parametrize("generic", [False, True])
def test_gemm_propagates_nan_and_inf(gpu, generic):
    """NaN and Inf propagate as IEEE arithmetic without skipping zeros gives (0 * Inf = NaN): the F2J zero skip in dgemm
    is a documented deviation.  Finite entries within the usual 1e-10 of (|A||B|)-scaled error."""
    rng = np.random.default_rng(111)
    m, n, k = 70, 50, 40
    A, B = rng.standard_normal((m, k)), rng.standard_normal((k, n))
    A[3, 5] = np.inf
    A[10, :] = 0.0
    A[10, 7] = -np.inf
    B[7, 4] = 0.0                                      # -Inf * 0 = NaN in C(10, 4)
    B[9, 11] = np.nan
    A[20, 30], A[20, 31] = np.inf, -np.inf            # +Inf and -Inf in one row: NaN where both meet nonzero B
    B[2, 40] = np.inf
    for ta in (0, 1):
        for tb in (0, 1):
            got = dgemm(gpu, A, B, ta, tb, generic=generic)
            want = _explicit_product(A, B)
            assert np.array_equal(_classes(got), _classes(want)), (ta, tb)
            fin = np.isfinite(want)
            scale = np.abs(np.where(np.isfinite(A), A, 0)) @ np.abs(np.where(np.isfinite(B), B, 0))
            assert (np.abs(got[fin] - want[fin]) / np.maximum(scale[fin], 1e-300)).max() <= 1e-10


@pytest.mark.parametrize("generic", [False, True])
def test_gemm_beta_zero_and_alpha_zero(gpu, generic):
    """beta = 0 never reads C (C pre-filled with NaN); alpha = 0 or K = 0 with beta = 0 writes exact +0.0."""
    rng = np.random.default_rng(121)
    A, B = rng.standard_normal((130, 70)), rng.standard_normal((70, 90))
    got = dgemm(gpu, A, B, generic=generic)            # C starts as NaN
    assert np.isfinite(got).all()
    assert identical(dgemm(gpu, A, B, alpha=0.0, generic=generic), np.zeros((130, 90)))
    assert identical(dgemm(gpu, np.zeros((130, 0)), np.zeros((0, 90)), generic=generic), np.zeros((130, 90)))


def test_int8_split_non_finite_rows_and_columns(gpu):
    """Rows of A / columns of B holding NaN or Inf: those entries of C are non-finite, of the class the DMMA kernel gives,
    and every other entry is bit-identical to the same product with the poisoned rows and columns set to zero (their
    digits no longer leak into, or poison, the rest)."""
    rng = np.random.default_rng(131)
    m, n, k = 300, 280, 260
    A, B = rng.random((m, k)) - 0.5, rng.random((k, n)) - 0.5
    C0 = rng.standard_normal((m, n))
    Ap, Bp = A.copy(), B.copy()
    Ap[4, 10], Ap[200, 0], Ap[201, 5], Ap[201, 6] = np.nan, np.inf, np.inf, -np.inf
    Bp[3, 7], Bp[100, 250] = -np.inf, np.nan
    bad_r, bad_c = [4, 200, 201], [7, 250]
    Az, Bz = Ap.copy(), Bp.copy()
    Az[bad_r, :] = 0.0
    Bz[:, bad_c] = 0.0
    poisoned = np.zeros((m, n), dtype=bool)
    poisoned[bad_r, :] = True
    poisoned[:, bad_c] = True
    for C0_ in (None, C0):
        got = split_gemm(gpu, Ap, Bp, C0=C0_)
        clean = split_gemm(gpu, Az, Bz, C0=C0_)
        native = dgemm(gpu, Ap, Bp, C0=C0_, beta=0.0 if C0_ is None else 1.0)
        assert np.array_equal(~np.isfinite(got), poisoned)
        assert np.array_equal(_classes(got), _classes(native))
        assert identical(got[~poisoned], clean[~poisoned])


def test_int8_split_fold_with_an_overflowing_scale(gpu):
    """A row [2^1000, 1], a column [2^20, 2^39]: rowmax * colmax = 2^1039 overflows, so the weight 2^ex of the low digit
    groups is +Inf although their int32 sums are 0.  The product is 2^1020 + 2^39, which rounds to 2^1020 and is exactly
    what the split represents (both leading digits are exact); forming 0 * Inf used to make it NaN."""
    m = n = k = 256
    A, B = np.zeros((m, k)), np.zeros((k, n))
    A[0, 0], A[0, 1] = p2(1000), 1.0
    B[0, 0], B[1, 0] = p2(20), p2(39)
    A[1:, :] = np.random.default_rng(141).random((m - 1, k))
    got = split_gemm(gpu, A, B)
    assert got[0, 0] == p2(1020)
    assert np.isfinite(got).all()


def test_jacobi_rejects_non_finite_at_once(gpu):
    """A NaN or Inf in G is an error before any sweep (it used to rotate for 30 sweeps and then report no convergence)."""
    import marlin_b200 as mb
    lib, ctx = gpu
    for bad in (np.nan, np.inf, -np.inf):
        G = np.eye(50)
        G[30, 4] = G[4, 30] = bad
        with pytest.raises(nat.MarlinArgumentError, match="NaN or Inf"):
            mb.SubMatrix(G).symmetricEigen()
        w = (C.c_double * 50)()
        sweeps = C.c_int32(-1)
        rc = lib.mb_block_syev(ctx, upload_mat(gpu, G), alloc(gpu, 50, 50), w, C.byref(sweeps))
        assert rc == nat.MB_ERR_INVALID_ARG and sweeps.value == 0, (rc, sweeps.value)


# ============================================================================== D. exact arithmetic: ties and integers
def tie_lu_case(n, m=None, seed=0):
    """A = L U with L unit lower triangular, entries in {-1, 0, 1}, and U integer with a power-of-two diagonal: every
    column is a tie between the rows with l = +-1 (|a| = |u_cc|), so partial pivoting with the first index winning keeps
    the identity permutation; every intermediate is an integer far below 2^53."""
    m = m or n
    rng = np.random.default_rng(seed)
    L = np.tril(rng.integers(-1, 2, size=(m, n)), -1).astype(float)
    L[np.arange(n), np.arange(n)] = 1.0
    U = np.triu(rng.integers(-3, 4, size=(n, n))).astype(float)
    U[np.arange(n), np.arange(n)] = np.where(rng.random(n) < 0.5, -1, 1) * np.exp2(rng.integers(0, 3, size=n))
    L[:, 0] = np.where(rng.random(m) < 0.5, -1.0, 1.0)         # column 0: a tie among all rows
    L[0, 0] = 1.0
    return L @ U, L, U


@pytest.mark.parametrize("shape", [(31, 31), (32, 32), (33, 33), (64, 64), (65, 65), (130, 130), (257, 257), (300, 130)])
def test_lu_ties_everywhere_bit_for_bit(gpu, shape):
    """Identity permutation, L and U bit for bit (integers below 2^53: exact in any order), across both levels of the
    panel's pivot reduction and the panel boundaries at 32 columns."""
    m, n = shape
    A, L, U = tie_lu_case(n, m, seed=m * 7 + n)
    assert np.abs(A).max() * n < 2 ** 40
    got, perm = lu_gpu(gpu, A)
    assert np.array_equal(perm, np.arange(m))
    assert equal_values(np.tril(got[:, :n], -1), np.tril(L, -1)) and equal_values(np.triu(got[:n]), U)


@pytest.mark.parametrize("n", [31, 32, 33, 40])
def test_lu_ties_permuted_rows_against_exact_restatement(gpu, n):
    """P L U with a sparse L (entries +-1, column 0 all +-1: every row ties there): the pivots and factors come from the
    exact dgetf2 restatement, which also checks that every value it forms, and every partial sum of every update in any
    order, is an fp64 number (so the GPU must match it bit for bit).  Eliminating in a permuted order can create
    multipliers like 1/3; the test takes the first of a fixed sequence of row orders whose elimination stays exact."""
    rng = np.random.default_rng(n)
    L = (np.tril(rng.integers(-1, 2, size=(n, n)), -1) * (rng.random((n, n)) < 0.05)).astype(float) + np.eye(n)
    L[:, 0] = np.where(rng.random(n) < 0.5, -1.0, 1.0)
    L[0, 0] = 1.0
    U = np.triu(rng.integers(-3, 4, size=(n, n))).astype(float)
    U[np.arange(n), np.arange(n)] = np.where(rng.random(n) < 0.5, -1, 1) * np.exp2(rng.integers(0, 3, size=n))
    A = L @ U
    rng = np.random.default_rng(1000 + n)
    for _ in range(60):
        PA = A[rng.permutation(n)]
        lu, ipiv, exact = eo.getf2_exact(PA)
        if exact:
            break
    assert exact, "no exact row order found"
    got, perm = lu_gpu(gpu, PA)
    assert np.array_equal(perm, eo.perm_from_ipiv(ipiv, n))
    assert equal_values(got, lu)


def test_lu_subnormal_pivots(gpu):
    """Pivots below DBL_MIN: dgetf2 divides instead of scaling by the reciprocal (which is +Inf there)."""
    t = p2(-1060)
    A = np.array([[4 * t, 1.0], [2 * t, 1.0]])
    got, perm = lu_gpu(gpu, A)
    assert np.array_equal(perm, [0, 1]) and equal_values(got, np.array([[4 * t, 1.0], [0.5, 0.5]]))
    # larger: column 0 of a tie case made subnormal (multiples of 2^-1070, pivot 8 2^-1070), L's first column k/8
    n = 40
    _, L, U = tie_lu_case(n, seed=3)
    rng = np.random.default_rng(4)
    L[1:, 0] = rng.integers(-8, 9, size=n - 1) / 8.0
    U[0, 0] = 8 * p2(-1070)
    A = L @ U
    lu, ipiv, exact = eo.getf2_exact(A)
    assert exact and np.array_equal(ipiv, np.arange(n))
    got, perm = lu_gpu(gpu, A)
    assert np.array_equal(perm, np.arange(n)) and equal_values(got, lu)


@pytest.mark.parametrize("n", [64, 65, 200])
def test_cholesky_integer_factor_bit_for_bit(gpu, n):
    """A = L L^T, L integer lower triangular with a positive diagonal: square roots of perfect squares and quotients with
    integer results are exact, partial sums are integers below 2^53."""
    rng = np.random.default_rng(n)
    L = np.tril(rng.integers(-2, 3, size=(n, n)), -1) + np.diag(rng.integers(1, 4, size=n))
    A = (L @ L.T).astype(float)
    assert np.array_equal(np.array(eo.cholesky_int(A)), L)
    assert equal_values(cholesky_gpu(gpu, A), L)


def _tree_triangle(n, rng, unit):
    """I - N with one entry +-1 per row below the diagonal (row i points at a parent p(i) < i): the inverse is a sum over
    unique paths, entries in {-1, 0, 1}; times a +-1 diagonal when not unit."""
    T = np.eye(n)
    for i in range(1, n):
        T[i, rng.integers(0, i)] = rng.choice([-1.0, 1.0])
    if not unit:
        T = T * np.where(rng.random(n) < 0.5, -1.0, 1.0)[:, None]
    return T


@pytest.mark.parametrize("n", [64, 130])
def test_trsm_and_inverse_on_unimodular_triangles(gpu, n):
    """Integer unimodular triangles: X = T^-1 B and T^-1 are integers, every partial sum below 2^53 (checked)."""
    lib, ctx = gpu
    rng = np.random.default_rng(n)
    for unit in (1, 0):
        T = _tree_triangle(n, rng, unit)
        Ti = np.round(np.linalg.inv(T))
        assert np.array_equal(Ti @ T, np.eye(n))     # integer inverse, exactly
        B = rng.integers(-5, 6, size=(n, 37)).astype(float)
        X = Ti @ B
        assert (np.abs(T) @ np.abs(X) + np.abs(B)).max() < 2 ** 53
        hb = upload_mat(gpu, B)
        nat.check(lib.mb_block_trsm(ctx, upload_mat(gpu, T), 1, unit, hb))
        assert equal_values(download(gpu, hb, n, 37), X), unit
        ho = alloc(gpu, n, n)
        nat.check(lib.mb_block_inverse(ctx, upload_mat(gpu, T), ho))
        assert equal_values(download(gpu, ho, n, n), Ti), unit


@pytest.mark.parametrize("cfg", [(16, 20), (24, 20), (48, 10)])
def test_jacobi_graded_matrices_relative_accuracy(cfg):
    """G = D M D, D = diag(2^-g i), M well conditioned with a unit diagonal.  Two-sided Jacobi with the relative stopping
    rule |g_pq| <= eps sqrt|g_pp| sqrt|g_qq| gives every eigenvalue to a relative error of about eps kappa(M)
    (Demmel-Veselic), the tiny ones included; the reference is mpmath with precision to spare.  Bound: 4 n eps kappa(M)."""
    import marlin_b200 as mb
    n, g = cfg
    rng = np.random.default_rng(n)
    S = rng.standard_normal((n, n)) / (2 * np.sqrt(n))
    M = np.eye(n) + (S + S.T) / 2
    np.fill_diagonal(M, 1.0)
    kappa = np.linalg.cond(M)
    d = np.exp2(-g * np.arange(n, dtype=float))
    G = d[:, None] * M * d[None, :]
    want = np.array(sorted(eo.eigvalsh_mp(G), key=lambda x: -abs(x)))
    w, _ = mb.SubMatrix(G).symmetricEigen()
    rel = np.abs(w - want) / np.abs(want)
    assert rel.max() <= 4 * n * EPS * kappa, (rel.max(), kappa)


def test_jacobi_ties_in_magnitude_keep_index_order():
    """Eigenvalues +-1 and repeated values: ordered by |w| descending, ties by index (the diagonal position)."""
    import marlin_b200 as mb
    d = np.array([1.0, -2.0, 1.0, 2.0, -1.0, 3.0, 2.0])
    w, V = mb.SubMatrix(np.diag(d)).symmetricEigen()
    order = sorted(range(len(d)), key=lambda i: (-abs(d[i]), i))
    assert identical(w, d[order])
    assert identical(V.toBreeze(), np.eye(len(d))[:, order])


# ============================================================================ E. views inside poisoned parents
SENTINEL = 12345.678


def _parent_with(X, ld, r0, c0, cols_total, fill=np.nan):
    """A column-major parent (ld x cols_total) filled with `fill`, X stored at (r0, c0): returns the flat parent and
    the element offset of the view."""
    P = np.full((ld, cols_total), fill)
    P[r0:r0 + X.shape[0], c0:c0 + X.shape[1]] = X
    return P, r0 + c0 * ld


def _view_of(gpu, X, trans=0, pad=(6, 4, 2, 2)):
    """X (logical) as a view with even ld and an aligned offset inside a NaN parent: the TMA path's requirements met.
    trans: X^T stored, is_transpose = 1."""
    S = X.T if trans else X
    ld = S.shape[0] + pad[0]
    P, off = _parent_with(S, ld, pad[2], pad[3], S.shape[1] + pad[1])
    t = cuda(P)
    return t, wrap(gpu, t, X.shape[0], X.shape[1], ld, off, trans)


def _out_view(gpu, rows, cols, pad=(4, 3, 2, 1)):
    ld = rows + pad[0]
    P, off = _parent_with(np.zeros((rows, cols)), ld, pad[2], pad[3], cols + pad[1], fill=SENTINEL)
    P[pad[2]:pad[2] + rows, pad[3]:pad[3] + cols] = np.nan
    t = cuda(P)
    return t, wrap(gpu, t, rows, cols, ld, off), (ld, off, P)


def _check_out(t, rows, cols, meta):
    ld, off, P = meta
    h = t.cpu().numpy()
    got = colmajor_host(t, rows, cols, ld, off)
    outside = h.reshape(-1).copy()
    for j in range(cols):
        outside[off + j * ld: off + j * ld + rows] = SENTINEL
    assert np.all(outside == SENTINEL), "a write outside the output view"
    return got


@pytest.mark.parametrize("ta", [0, 1])
@pytest.mark.parametrize("tb", [0, 1])
def test_gemm_views_in_poisoned_parents(gpu, ta, tb):
    """Operands as views of NaN-filled parents and C as a view of a sentinel-filled parent: the same bits as the call on
    packed copies (deterministic kernels, same path: even ld and aligned offsets either way), and no write outside C."""
    lib, ctx = gpu
    m, n, k = 130, 66, 98                       # ragged M against 128-row tiles; even leading dimensions for the copies
    rng = np.random.default_rng(151 + 2 * ta + tb)
    A, B = rng.standard_normal((m, k)), rng.standard_normal((k, n))
    C0 = rng.standard_normal((m, n))
    want = dgemm(gpu, A, B, ta, tb)
    want_acc = dgemm(gpu, A, B, ta, tb, C0=C0, beta=1.0)
    ta_, va = _view_of(gpu, A, ta)
    tb_, vb = _view_of(gpu, B, tb)
    tc, vc, meta = _out_view(gpu, m, n)
    nat.check(lib.mb_block_gemm(ctx, va, vb, vc, 0))
    sync(gpu)
    assert identical(_check_out(tc, m, n, meta), want)
    nat.check(lib.mb_block_copy(ctx, upload_mat(gpu, C0), vc))
    nat.check(lib.mb_block_gemm(ctx, va, vb, vc, 1))
    sync(gpu)
    assert identical(_check_out(tc, m, n, meta), want_acc)


def test_gramian_gemv_views_in_poisoned_parents(gpu):
    lib, ctx = gpu
    rng = np.random.default_rng(171)
    A = rng.standard_normal((300, 130))
    # Gramian
    hg = alloc(gpu, 130, 130)
    nat.check(lib.mb_block_gramian(ctx, upload_mat(gpu, A), hg))
    want = download(gpu, hg, 130, 130)
    _, va = _view_of(gpu, A)
    tg, vg, meta = _out_view(gpu, 130, 130)
    nat.check(lib.mb_block_gramian(ctx, va, vg))
    sync(gpu)
    assert identical(_check_out(tg, 130, 130, meta), want)
    # gemv, both orientations
    x = rng.standard_normal(130)
    for trans in (0, 1):
        X = A.T if trans else A
        rows = X.shape[0]
        xx = x if not trans else rng.standard_normal(300)
        hy = alloc(gpu, rows, 1)
        hx = upload_mat(gpu, xx[:, None])
        hA = upload_mat(gpu, A)
        if trans:
            v = nat.c_blk()
            nat.check(lib.mb_block_view_t(ctx, hA, C.byref(v)))
            hA = v
        nat.check(lib.mb_block_gemv(ctx, hA, hx, hy, 0))
        want = download(gpu, hy, rows, 1)
        _, vA = _view_of(gpu, X, trans)
        _, vx = _view_of(gpu, xx[:, None])
        ty, vy, meta = _out_view(gpu, rows, 1)
        nat.check(lib.mb_block_gemv(ctx, vA, vx, vy, 0))
        sync(gpu)
        assert identical(_check_out(ty, rows, 1, meta), want), trans


def test_factorization_views_in_poisoned_parents(gpu):
    """LU, Cholesky and trsm in place on views: the same bits as on packed blocks, the parent untouched outside."""
    lib, ctx = gpu
    rng = np.random.default_rng(181)
    n = 130
    A = rng.random((n, n)) - 0.5
    want, perm_want = lu_gpu(gpu, A)
    tA, vA, meta = _out_view(gpu, n, n)
    nat.check(lib.mb_block_copy(ctx, upload_mat(gpu, A), vA))
    perm = (C.c_int32 * n)()
    nat.check(lib.mb_block_lu(ctx, vA, perm))
    sync(gpu)
    assert identical(_check_out(tA, n, n, meta), want) and np.array_equal(perm[:], perm_want)
    G = rng.standard_normal((n, n))
    S = G @ G.T + n * np.eye(n)
    want = cholesky_gpu(gpu, S)
    tS, vS, meta = _out_view(gpu, n, n)
    nat.check(lib.mb_block_copy(ctx, upload_mat(gpu, S), vS))
    nat.check(lib.mb_block_cholesky(ctx, vS))
    sync(gpu)
    assert identical(_check_out(tS, n, n, meta), want)
    T = np.tril(rng.random((n, n)) - 0.5) + 4 * np.eye(n)
    B = rng.random((n, 50)) - 0.5
    hb = upload_mat(gpu, B)
    nat.check(lib.mb_block_trsm(ctx, upload_mat(gpu, T), 1, 0, hb))
    want = download(gpu, hb, n, 50)
    _, vT = _view_of(gpu, T)
    tB, vB, meta = _out_view(gpu, n, 50)
    nat.check(lib.mb_block_copy(ctx, upload_mat(gpu, B), vB))
    nat.check(lib.mb_block_trsm(ctx, vT, 1, 0, vB))
    sync(gpu)
    assert identical(_check_out(tB, n, 50, meta), want)

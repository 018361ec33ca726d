"""The exact-integer data of tests/test_gpu_fp64_exact.py, proved on the CPU: the generated products are exact in
float64, use the top of the 2^53 range, and a product just over the bound is refused."""
import numpy as np
import pytest

from tests import exact_gemm as xg

ALPHAS = [1.0, -3.0, 2.0 ** -4]
BETAS = [0.0, 1.0, -2.0]
KS = [1, 2, 3, 15, 16, 17, 95, 96, 97, 1000, 1030, 4096, 4097, 4099, 8192, 20000]


@pytest.mark.parametrize("alpha", ALPHAS)
@pytest.mark.parametrize("beta", BETAS)
def test_magnitudes_fill_the_significand(alpha, beta):
    for K in KS:
        amax, bmax, cmax = xg.magnitudes(K, alpha, beta)
        w = xg.worst_case(K, amax, bmax, alpha, beta, cmax)
        assert xg.TWO52 <= w <= xg.TWO53, (K, alpha, beta, w)
        assert (cmax > 0) == (beta != 0.0)
    for K in KS:
        amax = xg.magnitudes(K, square=True)[0]
        assert xg.TWO52 <= xg.worst_case(K, amax, amax) <= xg.TWO53, K


def test_magnitudes_of_the_named_cases():
    """K = 4099 keeps |a|, |b| near 2^20.5; K = 1 near 2^26.5; alpha = 2^-4 leaves the magnitudes of alpha = 1."""
    a, b, _ = xg.magnitudes(4099)
    assert 2 ** 20 <= a <= b < 2 ** 21
    a, b, _ = xg.magnitudes(1)
    assert 2 ** 26 <= a <= b < 2 ** 27
    assert xg.magnitudes(97, 2.0 ** -4) == xg.magnitudes(97)
    assert xg.unit_exponent(2.0 ** -4, -2.0) == 4 and xg.unit_exponent(-3.0, 1.0) == 0


@pytest.mark.parametrize("shape", [(1, 1, 1), (5, 1, 7), (2, 17, 3), (33, 97, 29), (64, 1000, 64), (130, 4099, 40),
                                   (3, 20000, 2)])
@pytest.mark.parametrize("alpha,beta", [(1.0, 0.0), (-3.0, 1.0), (2.0 ** -4, -2.0), (2.0 ** -4, 0.0)])
def test_float64_product_equals_int64_product(shape, alpha, beta):
    m, k, n = shape
    rng = np.random.default_rng(m + 7 * k + 13 * n)
    A, B, C0 = xg.operands(rng, m, k, n, alpha, beta)
    w = xg.check_bound(A, B, alpha, beta, C0)
    assert xg.TWO52 <= w <= xg.TWO53
    p = xg.unit_exponent(alpha, beta)
    ia, ib = int(alpha * 2 ** p), int(beta * 2 ** p)
    exact = ia * (A.astype(np.int64) @ B.astype(np.int64))             # in units of 2^-p; |.| <= 2^53 < 2^63
    if C0 is not None:
        exact = exact + ib * C0.astype(np.int64)
    ref = xg.reference(A, B, alpha, beta, C0)
    scaled = ref * 2.0 ** p
    assert np.array_equal(scaled, np.trunc(scaled))
    assert np.array_equal(scaled.astype(np.int64), exact)
    # result (0, 0) is the worst case itself: the top of the range is really used
    assert abs(int(exact[0, 0])) == w
    # signs are mixed, so other sums cancel
    if m * k * n > 1:
        assert (A < 0).any() and (A > 0).any() and (B < 0).any() and (B > 0).any()


def test_bound_check_refuses_products_over_2_53():
    A = np.array([[2.0 ** 26, 2.0 ** 26]])
    xg.check_bound(A, np.array([[2.0 ** 26], [2.0 ** 26]]))                          # exactly 2^53: exact
    with pytest.raises(AssertionError, match="exceeds 2"):
        xg.check_bound(A, np.array([[2.0 ** 26 + 1], [2.0 ** 26]]))                  # 2^53 + 2^27
    # one more k at the magnitudes chosen for K tips it over
    rng = np.random.default_rng(0)
    A, B, _ = xg.operands(rng, 4, 4099, 3)
    amax, bmax, _ = xg.magnitudes(4099)
    xg.check_bound(A, B)
    with pytest.raises(AssertionError):
        xg.check_bound(np.full((1, 4101), float(amax)), np.full((4101, 1), float(bmax)))
    # alpha = 2^-4 counts in units of 2^-4: an addend of 2^49 + 1 is 2^53 + 16 units with beta = 1
    small = np.full((1, 1), 2.0 ** 25)
    xg.check_bound(small, small, 2.0 ** -4, 1.0, np.full((1, 1), 2.0 ** 48))
    with pytest.raises(AssertionError):
        xg.check_bound(small, small, 2.0 ** -4, 1.0, np.full((1, 1), 2.0 ** 49 + 1))
    with pytest.raises(ValueError):
        xg.check_bound(np.full((1, 1), 0.5), small)


def test_report_locates_and_classifies():
    want = np.arange(300 * 260, dtype=np.float64).reshape(300, 260)
    got = want.copy()
    got[130:140, 200:210] = np.nan                                     # a tile never written
    got[299, 0] += 3.0                                                 # a wrong term
    msg = xg.report(got, want)
    assert "101 of 78000 elements wrong" in msg
    assert "rows 130..299, columns 0..209" in msg and "tiles 1..2 x 0..1" in msg
    assert "100 NaN (never written), 1 finite and off by 3..3, 1 by an integer" in msg
    with pytest.raises(AssertionError, match="never written"):
        xg.assert_exact(got, want, "case")
    xg.assert_exact(np.array([-0.0]), np.array([0.0]))                # -0.0 == +0.0 as numbers
    with pytest.raises(AssertionError):
        xg.assert_exact(np.array([np.nan]), np.array([np.nan]))         # NaN is never a right answer

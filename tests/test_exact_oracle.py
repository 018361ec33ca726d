"""Pins the exact references of tests/exact_oracle.py on the CPU: the dgetf2 restatement against LAPACK and hand-worked
tie and subnormal cases, the integer Cholesky, and the mpmath eigenvalues against LAPACK's."""
import numpy as np
import pytest
import scipy.linalg as sla

from tests import exact_oracle as eo


@pytest.mark.parametrize("shape", [(1, 1), (2, 2), (7, 7), (20, 20), (30, 12), (12, 30)])
def test_getf2_matches_lapack_on_tie_free_data(shape):
    """Random data has no ties, so the pivots must be LAPACK's exactly; the values are the exact rational LU rounded once,
    LAPACK's are rounded at every step: within 1e-12 relative to max|U| (small, well-conditioned matrices)."""
    m, n = shape
    rng = np.random.default_rng(m * 100 + n)
    A = rng.random((m, n)) - 0.5
    lu, ipiv, exact = eo.getf2_exact(A)
    assert exact == (shape == (1, 1))                  # generic data rounds as soon as there is an update
    P, L, U = sla.lu(A)
    k = min(m, n)
    perm = eo.perm_from_ipiv(ipiv, m)
    assert np.array_equal(P.T @ A, A[perm])            # the same row order as LAPACK's
    assert np.abs(np.tril(lu[:, :k], -1) + np.eye(m, k) - L).max() <= 1e-12
    assert np.abs(np.triu(lu[:k, :]) - U).max() <= 1e-12 * max(1.0, np.abs(U).max())
    if m == n:
        assert np.array_equal(ipiv, sla.lu_factor(A)[1])


def test_getf2_first_index_wins_ties():
    """Every column is a tie: |a| = 2 in rows 0 and 1 of column 0, then 1 and 1.  The first row wins each time."""
    A = np.array([[2.0, 1.0, 0.0], [-2.0, 1.0, 3.0], [2.0, 3.0, 1.0]])
    lu, ipiv, exact = eo.getf2_exact(A)
    assert exact and ipiv.tolist() == [0, 1, 2]
    # column 0: l = -1, 1; row 1 -> [0, 2, 3], row 2 -> [0, 2, 1]; column 1: |2| = |2|, row 1 wins, l = 1; u22 = 1 - 3
    want = np.array([[2.0, 1.0, 0.0], [-1.0, 2.0, 3.0], [1.0, 1.0, -2.0]])
    assert np.array_equal(lu, want)
    B = A[[2, 0, 1]]                                   # the same rows, permuted: still all ties
    lu2, ipiv2, exact2 = eo.getf2_exact(B)
    assert exact2 and ipiv2.tolist() == [0, 2, 2]
    perm = eo.perm_from_ipiv(ipiv2, 3)
    L = np.tril(lu2, -1) + np.eye(3)
    assert np.array_equal(L @ np.triu(lu2), B[perm])


def test_getf2_divides_by_a_subnormal_pivot():
    """[[4 t, 1], [2 t, 1]], t = 2^-1060: the pivot 2^-1058 is below sfmin, so dgetf2 divides: l = 0.5, u22 = 0.5.
    Its reciprocal (2^1058) would overflow."""
    t = 2.0 ** -1060
    A = np.array([[4 * t, 1.0], [2 * t, 1.0]])
    lu, ipiv, exact = eo.getf2_exact(A)
    assert exact and ipiv.tolist() == [0, 1]
    assert np.array_equal(lu, np.array([[4 * t, 1.0], [0.5, 0.5]]))
    # above sfmin the reciprocal is used: 1/3 is not an fp64 number, so the factorization of [[3, 1], [1, 1]] is not exact
    assert not eo.getf2_exact(np.array([[3.0, 1.0], [1.0, 1.0]]))[2]
    assert eo.getf2_exact(np.array([[4.0, 1.0], [1.0, 1.0]]))[2]


def test_getf2_exactness_bound():
    """Entries whose partial sums need more than 53 bits are not exact, even when every final value is an fp64 number."""
    A = np.array([[1.0, 2.0 ** 53], [1.0, 1.0]])
    assert not eo.getf2_exact(A)[2]
    assert eo.getf2_exact(np.array([[1.0, 2.0 ** 40], [1.0, 1.0]]))[2]


def test_cholesky_int():
    rng = np.random.default_rng(1)
    n = 30
    L = np.tril(rng.integers(-3, 4, size=(n, n)), -1) + np.diag(rng.integers(1, 5, size=n))
    A = L @ L.T
    assert np.array_equal(np.array(eo.cholesky_int(A)), L)
    with pytest.raises(ValueError):
        eo.cholesky_int(np.array([[2, 1], [1, 2]]))
    with pytest.raises(ValueError):
        eo.cholesky_int(np.array([[4, 1], [1, 2]]))          # 1/2 is not an integer


@pytest.mark.parametrize("n", [1, 2, 6, 15])
def test_mpmath_eigenvalues_match_lapack(n):
    """Unit-scale symmetric matrices: LAPACK is accurate to ~n eps ||G|| there, mpmath to 40 digits."""
    rng = np.random.default_rng(n)
    S = rng.standard_normal((n, n))
    G = S + S.T
    want = np.linalg.eigvalsh(G)
    got = np.array(eo.eigvalsh_mp(G))
    assert np.abs(got - want).max() <= 1e-13 * max(1.0, np.abs(want).max())


def test_mpmath_eigenvalues_of_a_graded_matrix():
    """G = D M D with D = diag(2^-20i): every eigenvalue is within a few eps kappa(M) of d_i^2 m_ii-ish; the mpmath
    reference must resolve the smallest one (2^-200 here) to full relative accuracy, which a norm-relative solver at 40
    digits would not.  Checked against the product of the eigenvalues, det(G) = det(M) prod d_i^2."""
    n = 6
    rng = np.random.default_rng(3)
    S = rng.standard_normal((n, n)) * 0.1
    M = np.eye(n) + (S + S.T) / 2
    np.fill_diagonal(M, 1.0)
    d = 2.0 ** (-20 * np.arange(n))
    G = d[:, None] * M * d[None, :]
    w = np.array(eo.eigvalsh_mp(G))
    assert np.all(w > 0)
    logdet = np.log(w).sum()
    want = np.linalg.slogdet(M)[1] + 2 * np.log(d).sum()
    assert abs(logdet - want) <= 1e-12 * abs(want)

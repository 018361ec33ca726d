"""Host logic of the Lanczos computeSVD overload, no GPU needed: the mode chooser mb_svd_plan against a chooser restated
here from the reference (:1557-1604, :1466-1468), and the projected eigensolver mb_eigs_projected against LAPACK."""
import ctypes as C

import numpy as np
import pytest

from marlin_b200 import _native as nat

CODES = {"local-svd": nat.MB_SVD_LOCAL_LAPACK, "local-eigs": nat.MB_SVD_LOCAL_ARPACK, "dist-eigs": nat.MB_SVD_DIST_ARPACK}


@pytest.fixture(scope="module")
def lib():
    return nat.load()


def plan(n: int, k: int, mode: str, max_iter: int) -> str:
    """The reference's chooser with the column cap only where G is formed."""
    if not (0 < k <= n):
        raise ValueError(f"Request up to n singular values but got k={k} and n={n}.")
    if mode == "auto":
        cm = ("local-eigs" if k < n // 3 else "local-svd") if (n < 100 or k > n // 2) else "dist-eigs"
    elif mode in CODES:
        cm = mode
    else:
        raise ValueError(f"Do not support mode {mode}.")
    if cm != "local-svd" and not k < n:
        raise ValueError(f"k must be smaller than n in {cm} mode but got k={k} and n={n}.")
    if cm != "dist-eigs" and n > 65535:
        raise ValueError(f"Argument with more than 65535 cols: {n}")
    if cm != "local-svd" and max_iter <= 0:
        raise ValueError("ARPACK returns non-zero info = -4 The maximum number of Arnoldi update iterations allowed must be "
                         "greater than zero. (Refer ARPACK user guide for details)")
    return cm


NS = (1, 2, 3, 5, 99, 100, 101, 300, 65535, 65536, 70000, 2 ** 31 - 1)
GRID = [(n, k, mode, it) for n in NS for k in sorted({0, 1, 2, n // 3, n // 2, n // 2 + 1, n - 1, n, n + 1} - {-1})
        for mode in ("auto", "local-svd", "local-eigs", "dist-eigs", "lanczos") for it in (300, 1, 0, -3)
        if 0 <= k <= 2 ** 31 - 1]


def test_svd_plan_matches_the_restated_chooser(lib):
    for n, k, mode, it in GRID:
        out = C.c_int32(-1)
        rc = lib.mb_svd_plan(n, k, mode.encode(), it, 1e-10, C.byref(out))
        try:
            want = plan(n, k, mode, it)
        except ValueError as e:
            assert rc == nat.MB_ERR_INVALID_ARG, (n, k, mode, it)
            assert lib.mb_last_error().decode() == str(e), (n, k, mode, it)
            continue
        assert rc == nat.MB_OK, (n, k, mode, it, lib.mb_last_error())
        assert out.value == CODES[want], (n, k, mode, it)


def test_svd_plan_keeps_the_cap_only_where_g_is_formed(lib):
    out = C.c_int32()
    assert lib.mb_svd_plan(70000, 5, b"dist-eigs", 300, 1e-10, C.byref(out)) == nat.MB_OK
    assert out.value == nat.MB_SVD_DIST_ARPACK
    for mode in (b"local-eigs", b"local-svd"):
        assert lib.mb_svd_plan(70000, 5, mode, 300, 1e-10, C.byref(out)) == nat.MB_ERR_INVALID_ARG
        assert lib.mb_last_error() == b"Argument with more than 65535 cols: 70000"
    # the older chooser still caps every mode
    assert lib.mb_svd_mode(70000, 5, b"dist-eigs", C.byref(out)) == nat.MB_ERR_INVALID_ARG
    assert lib.mb_svd_plan(2 ** 31 - 1, 10, b"auto", 300, 0.0, C.byref(out)) == nat.MB_OK
    assert out.value == nat.MB_SVD_DIST_ARPACK


def _projected(lib, T):
    n = T.shape[0]
    w = np.zeros(n)
    Z = np.zeros((n, n), order="F")
    Tf = np.asfortranarray(T)
    nat.check(lib.mb_eigs_projected(n, Tf.ctypes.data_as(nat.c_dp), w.ctypes.data_as(nat.c_dp), Z.ctypes.data_as(nat.c_dp)))
    return w, Z


def _check(T, w, Z):
    ref = np.sort(np.linalg.eigvalsh(T))[::-1]
    scale = max(np.abs(ref).max(), 1e-300)
    assert np.all(np.diff(w) <= 0)
    assert np.abs(w - ref).max() <= 1e-13 * scale
    assert np.abs(Z.T @ Z - np.eye(len(w))).max() <= 1e-13 * len(w)
    assert np.abs(T @ Z - Z * w).max() <= 1e-13 * scale * len(w)


@pytest.mark.parametrize("n", [1, 2, 3, 10, 40, 101])
def test_projected_tridiagonal(lib, n):
    rng = np.random.default_rng(n)
    for a, b in [(rng.standard_normal(n), rng.standard_normal(n - 1)),          # random
                 (np.full(n, 2.0), np.full(n - 1, -1.0)),                       # the 1-D Laplacian
                 (np.zeros(n), np.ones(n - 1)),                                 # zero diagonal
                 (np.arange(n, dtype=float) * 1e6, rng.standard_normal(n - 1) * 1e-6)]:
        T = np.diag(a) + np.diag(b, 1) + np.diag(b, -1)
        _check(T, *_projected(lib, T))


@pytest.mark.parametrize("n", [2, 5, 20, 60])
def test_projected_arrowhead(lib, n):
    """A thick restart leaves diag(theta) in the kept corner, an arrow in the next row and column, tridiagonal after."""
    rng = np.random.default_rng(100 + n)
    kk = max(1, n // 2)
    T = np.zeros((n, n))
    T[np.arange(kk), np.arange(kk)] = np.sort(rng.standard_normal(kk))[::-1] * 10
    T[kk - 1 if kk == n else kk, :kk] = T[:kk, kk - 1 if kk == n else kk] = rng.standard_normal(kk) * 1e-3
    for i in range(kk, n):
        T[i, i] = rng.standard_normal()
        if i + 1 < n:
            T[i, i + 1] = T[i + 1, i] = rng.standard_normal()
    T = (T + T.T) / 2
    _check(T, *_projected(lib, T))


def test_projected_reads_the_lower_triangle_and_rejects_non_finite(lib):
    T = np.array([[2.0, 99.0], [1.0, 3.0]])
    w, _ = _projected(lib, T)
    assert np.abs(w - np.linalg.eigvalsh(np.array([[2.0, 1.0], [1.0, 3.0]]))[::-1]).max() <= 1e-15 * 4
    T[1, 0] = np.nan
    w = np.zeros(2)
    Z = np.zeros(4)
    assert lib.mb_eigs_projected(2, np.asfortranarray(T).ctypes.data_as(nat.c_dp), w.ctypes.data_as(nat.c_dp),
                                 Z.ctypes.data_as(nat.c_dp)) == nat.MB_ERR_INVALID_ARG

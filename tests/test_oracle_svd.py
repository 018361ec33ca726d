"""The SVD oracle (tests/svd_oracle.py) against numpy, and the library's mode chooser / effective rank against the oracle
(pure host logic of the C ABI: no GPU needed)."""
import ctypes as C

import numpy as np
import pytest

from marlin_b200 import _native as nat
from tests import svd_oracle as so

# DistributedMatrixSuite.scala:375-388 (commented out in the reference)
SUITE_ROWS = [(0, [2.0, 0.0, 8.0, 6.0, 0.0]), (1, [1.0, 6.0, 0.0, 1.0, 7.0]), (2, [5.0, 0.0, 7.0, 4.0, 0.0]),
              (3, [7.0, 0.0, 8.0, 5.0, 0.0]), (4, [0.0, 10.0, 0.0, 0.0, 7.0])]


@pytest.fixture(scope="module")
def lib():
    return nat.load()


def test_suite_case_rounds_to_the_reference_values():
    U, s, V = so.compute_svd(SUITE_ROWS, 5, 3, compute_u=True)
    assert np.array_equal(np.round(s, 2), [17.92, 15.17, 3.56])
    A = np.array([r for _, r in SUITE_ROWS])
    Um = np.array([r for _, r in sorted(U)])
    assert np.allclose(Um * s @ V.T, A @ V @ V.T, atol=1e-10)


def test_gramian_is_dspr_and_triu_to_full():
    rng = np.random.default_rng(1)
    A = rng.standard_normal((37, 9))
    G = so.compute_gramian_matrix(list(enumerate(A)), 9, partitions=3)
    assert np.array_equal(G, G.T)
    assert np.abs(G - A.T @ A).max() <= 1e-12 * (np.abs(A.T) @ np.abs(A)).max()
    v = rng.standard_normal(9)
    assert np.allclose(so.multiply_gramian_matrix_by(list(enumerate(A)), v), A.T @ (A @ v))


@pytest.mark.parametrize("mode", ["local-svd", "local-eigs", "dist-eigs"])
def test_each_oracle_mode_agrees_with_numpy(mode):
    rng = np.random.default_rng(2)
    A = rng.standard_normal((200, 40))
    ref = np.linalg.svd(A, compute_uv=False)
    U, s, V = so.compute_svd(list(enumerate(A)), 40, 8, compute_u=True, mode=mode)
    assert np.allclose(s, ref[:8], rtol=1e-9)
    assert np.allclose(V.T @ V, np.eye(8), atol=1e-9)
    Um = np.array([r for _, r in sorted(U)])
    assert np.allclose(Um.T @ Um, np.eye(8), atol=1e-8)


GRID = [(n, k, mode) for n in (1, 2, 3, 5, 99, 100, 101, 300, 65535, 65536, 70000)
        for k in (-1, 0, 1, 2, 33, 34, 49, 50, 51, 99, 100, 101, 150, 151, 299, 300, 301)
        for mode in ("auto", "local-svd", "local-eigs", "dist-eigs", "lanczos")]


def test_svd_mode_matches_the_oracle(lib):
    codes = {"local-svd": nat.MB_SVD_LOCAL_LAPACK, "local-eigs": nat.MB_SVD_LOCAL_ARPACK, "dist-eigs": nat.MB_SVD_DIST_ARPACK}
    seen = set()
    for n, k, mode in GRID:
        out = C.c_int32(-1)
        rc = lib.mb_svd_mode(n, k, mode.encode(), C.byref(out))
        try:
            want = so.svd_mode(n, k, mode)
        except ValueError as e:
            assert rc == nat.MB_ERR_INVALID_ARG, (n, k, mode)
            assert lib.mb_last_error().decode() == str(e), (n, k, mode)
            seen.add(str(e).split(" ")[0])
            continue
        assert rc == nat.MB_OK and out.value == codes[want], (n, k, mode, want, out.value)
        seen.add(want)
    assert seen >= {"local-svd", "local-eigs", "dist-eigs", "Request", "Do", "k", "Argument"}


@pytest.mark.parametrize("rcond", [0.0, 1e-9, 1e-3, 0.5, 1.0, 2.0])
def test_svd_rank_matches_the_oracle(lib, rcond):
    rng = np.random.default_rng(3)
    for count in (0, 1, 5, 20):
        sig = np.sort(rng.random(count))[::-1].copy()
        if count > 3:
            sig[3] = sig[2]                              # ties count as kept (>= threshold)
        for k in (1, 3, 5, 20, 30):
            got = lib.mb_svd_rank(sig.ctypes.data_as(nat.c_dp), count, k, rcond)
            assert got == so.effective_rank(sig, k, rcond), (count, k, rcond)

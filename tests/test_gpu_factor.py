"""SURVEY 8 f4 tail at the C ABI: LU / Cholesky / inverse / triangular solve of one device block against LAPACK (scipy /
numpy: the same dgetrf / dpotrf / dgetri / dtrtrs family Breeze calls in matrix/DenseVecMatrix.scala:302,495,587).
Tolerances: pivot choices and permutations EXACT (partial pivoting is an index decision; generic random data has no ties);
factors and inverses within 1e-10 of LAPACK's, scaled by the magnitudes a backward-stable factorization is judged by;
size-independent properties (P A = L U, L L^T = A, A A^-1 = I) at the largest sizes."""
import ctypes as C

import numpy as np
import pytest
import scipy.linalg as sla

from marlin_b200 import _native as nat
from tests.harness import gpu  # noqa: F401  (a fixture)
from tests.test_gpu_cabi import alloc, download, upload_mat

pytestmark = pytest.mark.gpu


def lu_gpu(gpu, A):
    lib, ctx = gpu
    h = upload_mat(gpu, A)
    perm = (C.c_int32 * A.shape[0])()
    nat.check(lib.mb_block_lu(ctx, h, perm))
    out = download(gpu, h, *A.shape)
    nat.check(lib.mb_block_free(ctx, h))
    return out, np.array(perm[:], dtype=np.int64)


@pytest.mark.parametrize("shape", [(1, 1), (2, 2), (5, 5), (33, 33), (64, 64), (100, 100), (257, 257), (1000, 1000),
                                   (300, 200), (200, 300), (2050, 2050)])
def test_lu_matches_lapack(gpu, shape):
    m, n = shape
    rng = np.random.default_rng(m * 31 + n)
    A = rng.random((m, n)) - 0.5
    got, perm = lu_gpu(gpu, A)
    lu, piv = sla.lu_factor(A) if m == n else (None, None)
    k = min(m, n)
    L = np.tril(got[:, :k], -1) + np.eye(m, k)
    U = np.triu(got[:k, :])
    # P A = L U, to backward-error accuracy
    resid = np.abs(A[perm] - L @ U).max() / (np.abs(L) @ np.abs(U)).max()
    assert resid <= 1e-13, resid
    assert sorted(perm.tolist()) == list(range(m))
    if m == n:
        want = np.arange(m)
        for i, p in enumerate(piv):                       # the reference's pArray construction (:303-308)
            want[i], want[p] = want[p], want[i]
        assert np.array_equal(perm, want)                 # the same pivot rows as dgetrf
        assert np.abs(got - lu).max() <= 1e-10 * max(1.0, np.abs(lu).max())


def test_lu_transposed_and_sliced_views(gpu):
    lib, ctx = gpu
    rng = np.random.default_rng(5)
    big = rng.random((300, 280)) - 0.5
    hb = upload_mat(gpu, big)
    v = nat.c_blk()
    nat.check(lib.mb_block_slice(ctx, hb, 10, 210, 20, 220, C.byref(v)))           # 200 x 200 view, ld = 300
    vt = nat.c_blk()
    nat.check(lib.mb_block_view_t(ctx, v, C.byref(vt)))                             # its transpose, no copy
    perm = (C.c_int32 * 200)()
    nat.check(lib.mb_block_lu(ctx, vt, perm))
    got = download(gpu, hb, 300, 280)[10:210, 20:220].T
    A = big[10:210, 20:220].T
    p = np.array(perm[:])
    L, U = np.tril(got, -1) + np.eye(200), np.triu(got)
    assert np.abs(A[p] - L @ U).max() <= 1e-13 * (np.abs(L) @ np.abs(U)).max()
    rest = download(gpu, hb, 300, 280)
    rest[10:210, 20:220] = big[10:210, 20:220]
    assert np.array_equal(rest, big)                                                # nothing outside the view was touched


@pytest.mark.parametrize("n", [1, 3, 64, 65, 130, 777, 2048])
def test_cholesky_matches_lapack(gpu, n):
    lib, ctx = gpu
    rng = np.random.default_rng(n)
    G = rng.random((n, n)) - 0.5
    A = G @ G.T + n * np.eye(n)
    h = upload_mat(gpu, A)
    nat.check(lib.mb_block_cholesky(ctx, h))
    L = download(gpu, h, n, n)
    want = np.linalg.cholesky(A)
    assert np.array_equal(np.triu(L, 1), np.zeros((n, n)))                         # Breeze `cholesky`: zeros above the diagonal
    assert np.abs(L - want).max() <= 1e-10 * np.abs(want).max()
    assert np.abs(L @ L.T - A).max() <= 1e-13 * np.abs(A).max() * max(1, n // 64)


def test_cholesky_rejects_indefinite(gpu):
    lib, ctx = gpu
    A = np.eye(40)
    A[17, 17] = -1.0
    h = upload_mat(gpu, A)
    rc = lib.mb_block_cholesky(ctx, h)
    assert rc == nat.MB_ERR_CUDA and b"positive definite" in lib.mb_last_error()


@pytest.mark.parametrize("n", [1, 3, 50, 64, 129, 500, 1536])
def test_inverse_matches_lapack(gpu, n):
    lib, ctx = gpu
    rng = np.random.default_rng(100 + n)
    A = rng.random((n, n)) - 0.5 + (2.0 if n > 1 else 1.0) * np.eye(n)
    h, o = upload_mat(gpu, A), alloc(gpu, n, n)
    nat.check(lib.mb_block_inverse(ctx, h, o))
    got = download(gpu, o, n, n)
    want = np.linalg.inv(A)
    assert np.abs(got - want).max() <= 1e-10 * np.abs(want).max()
    assert np.abs(A @ got - np.eye(n)).max() <= 1e-10


def test_inverse_suite_golden_and_singular(gpu):
    """DistributedMatrixSuite.scala:340-352: the inverse of the 3 x 3 exchange matrix is itself, exactly."""
    lib, ctx = gpu
    J = np.array([[0.0, 0.0, 1.0], [0.0, 1.0, 0.0], [1.0, 0.0, 0.0]])
    h, o = upload_mat(gpu, J), alloc(gpu, 3, 3)
    nat.check(lib.mb_block_inverse(ctx, h, o))
    assert np.array_equal(download(gpu, o, 3, 3), J)
    S = np.ones((4, 4))
    h, o = upload_mat(gpu, S), alloc(gpu, 4, 4)
    assert lib.mb_block_inverse(ctx, h, o) == nat.MB_ERR_CUDA and b"singular" in lib.mb_last_error()
    h2, o2 = upload_mat(gpu, np.ones((3, 4))), alloc(gpu, 3, 4)
    assert lib.mb_block_inverse(ctx, h2, o2) == nat.MB_ERR_DIM_MISMATCH


@pytest.mark.parametrize("case", [(40, 7, True, True), (64, 130, True, False), (200, 333, False, False), (1100, 260, True, True),
                                  (513, 513, False, True)])
def test_trsm_matches_lapack(gpu, case):
    lib, ctx = gpu
    t, nrhs, lower, unit = case
    rng = np.random.default_rng(t + nrhs)
    T = rng.random((t, t)) - 0.5 + 4.0 * np.eye(t)
    T = np.tril(T) if lower else np.triu(T)
    B = rng.random((t, nrhs)) - 0.5
    ht, hb = upload_mat(gpu, T), upload_mat(gpu, B)
    nat.check(lib.mb_block_trsm(ctx, ht, int(lower), int(unit), hb))
    got = download(gpu, hb, t, nrhs)
    want = sla.solve_triangular(T, B, lower=lower, unit_diagonal=unit)
    assert np.abs(got - want).max() <= 1e-10 * max(1.0, np.abs(want).max())
    # right-side solve X T = B through transposed views: T^T X^T = B^T
    B2 = rng.random((nrhs, t)) - 0.5
    hb2 = upload_mat(gpu, B2)
    tt, bt = nat.c_blk(), nat.c_blk()
    nat.check(lib.mb_block_view_t(ctx, ht, C.byref(tt)))
    nat.check(lib.mb_block_view_t(ctx, hb2, C.byref(bt)))
    nat.check(lib.mb_block_trsm(ctx, tt, int(not lower), int(unit), bt))
    got2 = download(gpu, hb2, nrhs, t)
    want2 = sla.solve_triangular(T.T, B2.T, lower=not lower, unit_diagonal=unit).T
    assert np.abs(got2 - want2).max() <= 1e-10 * max(1.0, np.abs(want2).max())


def test_factorizations_full_size_properties(gpu):
    """4096^2 (local-mode sizes go up to 6000 in the reference, :290): residuals only — no LAPACK run needed."""
    lib, ctx = gpu
    n = 4096
    rng = np.random.default_rng(9)
    A = rng.random((n, n)) - 0.5
    got, perm = lu_gpu(gpu, A)
    L, U = np.tril(got, -1) + np.eye(n), np.triu(got)
    assert np.abs(L).max() <= 1.0 + 1e-12                                          # partial pivoting: |l_ij| <= 1
    x = rng.random(n)
    assert np.abs(A[perm] @ x - L @ (U @ x)).max() <= 1e-10 * (np.abs(L) @ (np.abs(U) @ np.abs(x))).max()
    Ad = A + 64.0 * np.eye(n)
    h, o = upload_mat(gpu, Ad), alloc(gpu, n, n)
    nat.check(lib.mb_block_inverse(ctx, h, o))
    inv = download(gpu, o, n, n)
    assert np.abs(Ad @ (inv @ x) - x).max() <= 1e-10
    S = A @ A.T + n * np.eye(n)
    hs = upload_mat(gpu, S)
    nat.check(lib.mb_block_cholesky(ctx, hs))
    Lc = download(gpu, hs, n, n)
    assert np.abs(Lc @ (Lc.T @ x) - S @ x).max() <= 1e-10 * np.abs(S @ x).max()

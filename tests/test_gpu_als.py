"""CoordinateMatrix.ALS on the GPU: the assembly-only instance (mb_als_normal_equations) bit for bit against the oracle's
ordered sums (tests/als_oracle.py), the fused Cholesky solve (mb_als_update) within a kappa(A)-scaled bound, whole runs
against the oracle half-step by half-step, the initial factors, run-to-run and two-rank determinism, the errors, and a
MovieLens-20M-shaped run."""
import ctypes as C
import os
import socket
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import scipy.linalg

from tests import als_oracle as ao

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
U_ = 2.0 ** -53


def _nat():
    from marlin_b200 import _native as nat
    return nat


def _rows_block(X):
    """A row-major device view of the host array X (n x r), as the factor matrices are held."""
    import torch
    import marlin_b200 as mb
    t = torch.from_numpy(np.ascontiguousarray(X, np.float64).reshape(-1)).cuda()
    return mb.SubMatrix(buf=t, rows=X.shape[0], cols=X.shape[1], ld=X.shape[1], is_transpose=True)


def _links(ent, partner, vals, nb, npb):
    from marlin_b200.matrix.coordinate_matrix import _Links
    return _Links(ent, partner, vals, nb, npb)


def _gpu_assemble(L, Y, lam, implicit=False, alpha=1.0, yty=None):
    import torch
    import marlin_b200 as mb
    nat = _nat()
    rt = mb.Runtime.get()
    rt.sync_stream()
    r = Y.shape[1]
    side, keep = L.to_device(rt.device)
    A = torch.full((L.n * (r * (r + 1) // 2),), float("nan"), dtype=torch.float64, device=rt.device)
    b = torch.full((L.n * r,), float("nan"), dtype=torch.float64, device=rt.device)
    Yb = _rows_block(Y)
    G = _rows_block(yty) if yty is not None else None
    nat.check(rt.lib.mb_als_normal_equations(rt.ctx, C.byref(side), Yb.handle(), lam, alpha, int(implicit),
                                             G.handle() if G is not None else None, C.c_void_p(A.data_ptr()),
                                             C.c_void_p(b.data_ptr())))
    return A.cpu().numpy().reshape(L.n, -1), b.cpu().numpy().reshape(L.n, r)


def _gpu_update(L, Y, lam, implicit=False, alpha=1.0, yty=None):
    import marlin_b200 as mb
    nat = _nat()
    rt = mb.Runtime.get()
    rt.sync_stream()
    side, keep = L.to_device(rt.device)
    Xb = _rows_block(np.full((L.n, Y.shape[1]), np.nan))
    Yb = _rows_block(Y)                      # held until the call returns: the handle does not own the buffer
    G = _rows_block(yty) if yty is not None else None
    nat.check(rt.lib.mb_als_update(rt.ctx, C.byref(side), Yb.handle(), lam, alpha, int(implicit),
                                   G.handle() if G is not None else None, Xb.handle()))
    return Xb.toBreeze()


def _data(nu, npr, nnz, seed, heavy=0, signed=False):
    rng = np.random.default_rng(seed)
    rows = rng.integers(0, nu, nnz)
    cols = rng.integers(0, npr, nnz)
    if heavy:
        rows = np.concatenate([rows, np.full(heavy, 3)])
        cols = np.concatenate([cols, rng.integers(0, npr, heavy)])
    rows = np.concatenate([rows, rows[:50]])                         # duplicated (row, col) entries
    cols = np.concatenate([cols, cols[:50]])
    lo = -3.0 if signed else 0.5
    vals = rng.uniform(lo, 5.0, len(rows)).astype(np.float32)
    return rows, cols, vals


def _solve_bound(Ap, b, r):
    """x from the oracle's exact A: cho_solve and inv(A) @ b, and the bound 16 r kappa(A) u max|x| the device's x must meet."""
    M = ao.full(Ap, r)
    x_inv = scipy.linalg.inv(M) @ b
    x_cho = scipy.linalg.cho_solve(scipy.linalg.cho_factor(M, lower=True), b)
    kappa = np.linalg.cond(M)
    return x_inv, x_cho, 16 * r * kappa * U_ * np.abs(x_cho).max()


@pytest.mark.parametrize("rank,npb", [(1, 1), (2, 3), (7, 10), (10, 3), (31, 1), (32, 10), (33, 3), (64, 10), (100, 1), (128, 3)])
def test_assembly_exact(rank, npb):
    rows, cols, vals = _data(60, 80, 2500, rank * 7 + npb, heavy=10000 if rank in (10, 33) else 0)
    rows = np.concatenate([rows, [1000]])                             # a user with a single rating
    cols = np.concatenate([cols, [79]])
    vals = np.concatenate([vals, np.array([2.7], np.float32)])
    L = _links(rows, cols, vals, 4, npb)
    Y = np.random.default_rng(rank).standard_normal((len(np.unique(cols)), rank)) * 0.7
    A, b = _gpu_assemble(L, Y, 0.037)
    A0, b0 = ao.assemble(ao.links(rows, cols, vals, 4, npb), Y, 0.037)
    assert np.array_equal(A.view(np.int64), A0.view(np.int64))
    assert np.array_equal(b.view(np.int64), b0.view(np.int64))


@pytest.mark.parametrize("rank", [3, 10, 40])
def test_assembly_exact_implicit(rank):
    rows, cols, vals = _data(50, 70, 3000, rank, signed=True)
    L = _links(rows, cols, vals, 3, 10)
    rng = np.random.default_rng(rank)
    Y = rng.standard_normal((len(np.unique(cols)), rank))
    yty = ao.gramian(rng.standard_normal((40, rank)))
    yty = (yty + yty.T) / 2
    A, b = _gpu_assemble(L, Y, 0.01, implicit=True, alpha=0.37, yty=yty)
    A0, b0 = ao.assemble(ao.links(rows, cols, vals, 3, 10), Y, 0.01, implicit=True, alpha=0.37, yty=yty)
    assert np.array_equal(A.view(np.int64), A0.view(np.int64))
    assert np.array_equal(b.view(np.int64), b0.view(np.int64))


@pytest.mark.parametrize("rank", [1, 10, 32, 33, 64, 128])
def test_solve_within_bound(rank):
    rows, cols, vals = _data(40, 300, 4000, rank + 1)
    L = _links(rows, cols, vals, 3, 4)
    Y = np.abs(np.random.default_rng(rank).standard_normal((len(np.unique(cols)), rank)))
    X = _gpu_update(L, Y, 0.05)
    A0, b0 = ao.assemble(ao.links(rows, cols, vals, 3, 4), Y, 0.05)
    for p in range(L.n):
        x_inv, x_cho, bound = _solve_bound(A0[p], b0[p], rank)
        assert np.abs(X[p] - x_cho).max() <= bound, p
        assert np.abs(X[p] - x_inv).max() <= bound, p


@pytest.mark.parametrize("implicit", [False, True])
def test_update_host_matches_device_update(implicit):
    """mb_als_update_host (host arrays, the JVM's updateBlock) gives the device entry's rows bit for bit."""
    import marlin_b200 as mb
    nat = _nat()
    rows, cols, vals = _data(30, 40, 900, 6, signed=implicit)
    L = _links(rows, cols, vals, 3, 2)
    rank = 9
    Y = np.abs(np.random.default_rng(2).standard_normal((len(np.unique(cols)), rank)))
    yty = np.ascontiguousarray(Y.T @ Y) if implicit else None
    want = _gpu_update(L, Y, 0.1, implicit, 0.5, yty)
    rt = mb.Runtime.get()
    X = np.zeros((L.n, rank))
    ptr = lambda a: C.c_void_p(a.ctypes.data) if a is not None else None
    ids, off = np.ascontiguousarray(L.ids), np.ascontiguousarray(L.offsets)
    nat.check(rt.lib.mb_als_update_host(rt.ctx, rank, Y.shape[0], ptr(Y), L.n, ptr(ids), ptr(off), ptr(L.partners),
                                        ptr(L.ratings), 0.1, 0.5, int(implicit), ptr(yty), ptr(X)))
    assert np.array_equal(X, want)


def _gpu_als(rows, cols, vals, *args, **kw):
    import marlin_b200 as mb
    U, P = mb.CoordinateMatrix((rows, cols, vals)).ALS(*args, **kw)
    return U.ids, U.data.toBreeze(), P.ids, P.data.toBreeze()


def test_initial_factors_bit_identical():
    rows, cols, vals = _data(70, 50, 900, 3)
    uid, U, pid, P = _gpu_als(rows, cols, vals, 17, 0, 0.1, 4, 6, seed=-5)
    oid, U0, qid, P0 = ao.als(rows, cols, vals, 17, 0, 0.1, 4, 6, seed=-5)
    assert np.array_equal(uid, oid) and np.array_equal(pid, qid)
    assert np.array_equal(U, U0) and np.array_equal(P, P0)


@pytest.mark.parametrize("implicit", [False, True])
def test_half_steps_against_oracle(implicit):
    """Each half-step of the device run against the oracle fed that half-step's device input (errors never compound)."""
    rows, cols, vals = _data(90, 60, 2500, 8, signed=implicit)
    rank, lam, alpha = 6, 0.08, 0.9
    users, products = ao.links(rows, cols, vals, 5, 4), ao.links(cols, rows, vals, 4, 5)
    prev_U = ao.init_factors(users, 13, 0, rank)
    for it in range(1, 4):
        _, U, _, P = _gpu_als(rows, cols, vals, rank, it, lam, 5, 4, implicit, alpha, seed=13)
        for L, Y, X in ((products, prev_U, P), (users, P, U)):
            A0, b0 = ao.assemble(L, Y, lam, implicit=implicit, alpha=alpha, yty=ao.gramian(Y) if implicit else None)
            for p in range(len(L.ids)):
                x_inv, x_cho, bound = _solve_bound(A0[p], b0[p], rank)
                # implicit: the device's YtY is a DMMA Gramian, the oracle's a numpy product; allow their difference
                tol = bound + (64 * rank * U_ * np.abs(Y).sum(0).max() ** 2 * np.abs(x_cho).max()
                               * np.linalg.norm(scipy.linalg.inv(ao.full(A0[p], rank)), 2) if implicit else 0.0)
                assert np.abs(X[p] - x_cho).max() <= tol, (it, p)
        prev_U = U


def test_run_to_run_bit_identical():
    rows, cols, vals = _data(200, 150, 8000, 4)
    a = _gpu_als(rows, cols, vals, 20, 2, 0.05, 7, 3, seed=1)
    b = _gpu_als(rows, cols, vals, 20, 2, 0.05, 7, 3, seed=1)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def test_two_ranks_bit_identical_to_one(tmp_path):
    sys.path.insert(0, str(ROOT / "tests"))
    import als_gpu_worker as w
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    env = dict(os.environ, ALS_WORKER_OUT=str(tmp_path / "f"))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), str(ROOT / "tests" / "als_gpu_worker.py")]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900, env=env)
    assert out.returncode == 0, out.stdout[-4000:]
    for r in range(2):
        assert f"rank {r} singular raised" in out.stdout and f"rank {r} duplicate raised" in out.stdout
    rows, cols, vals = w.data()
    # the ranks' entries are gathered in rank order, which is the input order (duplicates included) of the one-rank run
    order = np.concatenate([np.flatnonzero(np.arange(len(rows)) % 2 == r) for r in range(2)])
    rows, cols, vals = rows[order], cols[order], vals[order]
    for implicit in (False, True):
        uid, U, pid, P = _gpu_als(rows, cols, vals, 12, 2, 0.05, 5, 3, implicit, 0.7, seed=99)
        parts = [np.load(str(tmp_path / f"f.{int(implicit)}.{r}.npz")) for r in range(2)]
        for ids, X, key in ((uid, U, "U"), (pid, P, "P")):
            got_ids = np.concatenate([p[("u" if key == "U" else "p") + "id"] for p in parts])
            got = np.concatenate([p[key] for p in parts])
            order = np.argsort(got_ids)
            assert np.array_equal(got_ids[order], np.sort(ids))
            assert np.array_equal(got[order], X[np.argsort(ids)])


def test_errors():
    import marlin_b200 as mb
    nat = _nat()
    rows, cols, vals = _data(10, 10, 50, 0)
    m = mb.CoordinateMatrix((rows, cols, vals))
    with pytest.raises(nat.MarlinArgumentError) as e:
        m.ALS(129, 1, seed=0)
    assert e.value.code == nat.MB_ERR_UNSUPPORTED
    with pytest.raises(nat.MarlinArgumentError) as e:
        m.ALS(4, 1, -0.5, seed=0)
    assert e.value.code == nat.MB_ERR_INVALID_ARG
    with pytest.raises(nat.MarlinError, match="empty collection"):
        mb.CoordinateMatrix([]).ALS(4, 1, seed=0)
    # C ABI checks as well
    L = _links(rows, cols, vals, 2, 2)
    with pytest.raises(nat.MarlinArgumentError) as e:
        _gpu_update(L, np.ones((len(np.unique(cols)), 129)), 0.1)
    assert e.value.code == nat.MB_ERR_UNSUPPORTED
    with pytest.raises(nat.MarlinArgumentError):
        _gpu_update(L, np.ones((len(np.unique(cols)), 3)), -1.0)


def test_not_positive_definite_names_lowest_entity():
    # lambda = 0, rank 2: users 7 and 4 rate only product 0 whose factor is (1, 0) -> the second pivot is exactly 0
    nat = _nat()
    rows = np.array([7, 4, 9, 9])
    cols = np.array([0, 0, 0, 1])
    vals = np.array([1, 2, 3, 4], np.float32)
    L = _links(rows, cols, vals, 3, 1)
    Y = np.array([[1.0, 0.0], [0.0, 1.0]])
    with pytest.raises(nat.MarlinError, match="entity 4 are not positive definite"):
        _gpu_update(L, Y, 0.0)


def test_to_dense_vec_matrix():
    import marlin_b200 as mb
    nat = _nat()
    m = mb.CoordinateMatrix([((0, 1), 2.5), ((3, 0), -1.0), ((3, 4), 7.0)])
    d = m.toDenseVecMatrix()
    assert list(d.ids) == [0, 3]
    assert np.array_equal(d.toBreeze(), m.toBreeze())
    dup = mb.CoordinateMatrix([((0, 1), 2.5), ((0, 1), 1.0)])
    with pytest.raises(nat.MarlinArgumentError, match=r"requirement failed: Found duplicate indices: 1\."):
        dup.toDenseVecMatrix()


def _movielens_shape(seed):
    """138493 users x 26744 items, 20M ratings, power-law activity on both sides, half-star ratings."""
    rng = np.random.default_rng(seed)
    nu, ni, nnz = 138493, 26744, 20_000_000
    pu = 1.0 / np.arange(1, nu + 1) ** 0.6
    pi = 1.0 / np.arange(1, ni + 1) ** 0.9
    rows = rng.permutation(nu)[rng.choice(nu, nnz, p=pu / pu.sum())]
    cols = rng.permutation(ni)[rng.choice(ni, nnz, p=pi / pi.sum())]
    vals = (rng.integers(1, 11, nnz) / 2.0).astype(np.float32)
    return rows, cols, vals


@pytest.mark.parametrize("rank", [10, 50])
def test_movielens_20m_shape(rank):
    rows, cols, vals = _movielens_shape(2024)
    uid, U, pid, P = _gpu_als(rows, cols, vals, rank, 1, 0.05, 10, 10, seed=3)
    users, products = ao.links(rows, cols, vals, 10, 10), ao.links(cols, rows, vals, 10, 10)
    assert np.array_equal(uid, users.ids)
    counts = np.diff(users.offsets)
    assert counts.max() >= 10_000
    sample = np.unique(np.concatenate([users.work[:5], np.random.default_rng(0).choice(len(uid), 995, replace=False)]))
    U0 = ao.init_factors(users, 3, 0, rank)
    psample = np.unique(np.concatenate([products.work[:5], np.random.default_rng(1).choice(len(pid), 300, replace=False)]))
    for L, Y, X, pos in ((products, U0, P, psample), (users, P, U, sample)):
        A0, b0 = ao.assemble(L, Y, 0.05, positions=pos)
        for k, p in enumerate(pos):
            x_inv, x_cho, bound = _solve_bound(A0[k], b0[k], rank)
            assert np.abs(X[p] - x_cho).max() <= bound, p

"""computeSVD's Lanczos path on the GPU: the one-pass A^T (A x) kernel (mb_block_gram_matvec), the restarted Lanczos solver
behind mb_eigs_*, and the computeSVD(k, computeU, rCond, mode, maxIter=, tol=) overload on one and two ranks."""
import ctypes as C
import os
import socket
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from tests import svd_oracle as so

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
EPS = np.finfo(np.float64).eps / 2


@pytest.fixture(scope="module")
def M():
    import marlin_b200 as mb
    mb.Runtime.get()
    return mb


def _rowshard(M, A, ld=None, offset=0):
    """A (m x n) as a row shard: row r at offset + r * ld of a device buffer."""
    import torch
    m, n = A.shape
    ld = max(1, n) if ld is None else ld
    host = np.full(offset + max(m, 1) * ld, 7.5)
    for r in range(m):
        host[offset + r * ld: offset + r * ld + n] = A[r]
    return M.SubMatrix(buf=torch.from_numpy(host).cuda(), rows=m, cols=n, ld=ld, offset=offset, is_transpose=True)


def _vec(M, x):
    return M.SubMatrix(np.asarray(x, dtype=np.float64).reshape(-1, 1))


def _gmv(M, blk, x, y0=None, accumulate=False):
    from marlin_b200 import _native as nat
    rt = M.Runtime.get()
    rt.sync_stream()
    n = blk.cols
    xv, y = _vec(M, x), _vec(M, np.zeros(n) if y0 is None else y0)       # held: a handle lives as long as its SubMatrix
    nat.check(rt.lib.mb_block_gram_matvec(rt.ctx, blk.handle(), xv.handle(), y.handle(), int(accumulate)))
    return y.toBreeze().reshape(-1)


def _exact_shapes():
    for n in (1, 2, 127, 128, 129, 1024, 1500, 4097, 70000):
        for m in (0, 1, 31, 33, 100000):
            if m * n <= 2 ** 28:
                yield m, n


# --------------------------------------------------------------------------------------------------- the kernel
@pytest.mark.parametrize("m,n", list(_exact_shapes()))
def test_exact_integers(M, m, n):
    rng = np.random.default_rng(m * 131 + n)
    A = rng.integers(-3, 4, (m, n)).astype(np.float64)
    x = rng.integers(-3, 4, n).astype(np.float64)
    Ai = A.astype(np.int64)
    want = (Ai.T @ (Ai @ x.astype(np.int64))).astype(np.float64)
    views = [("row shard", lambda: _rowshard(M, A))]
    if m * n <= 2 ** 22:
        views += [("odd ld, offset", lambda: _rowshard(M, A, ld=n + 3, offset=1)), ("column-major", lambda: M.SubMatrix(A))]
    for name, make in views:
        got = _gmv(M, make(), x)
        assert np.array_equal(got, want), (m, n, name)


@pytest.mark.parametrize("m,n", [(3000, 300), (257, 5118), (257, 5119), (100, 20000), (1, 131072)])
def test_random_data_bound_accumulate_and_repeat(M, m, n):
    rng = np.random.default_rng(m + n)
    A = rng.standard_normal((m, n))
    x = rng.standard_normal(n)
    blk = _rowshard(M, A, ld=n + 1, offset=1)
    got = _gmv(M, blk, x)
    ref = A.T @ (A @ x)
    bound = 2 * (n + m) * EPS * (np.abs(A).T @ (np.abs(A) @ np.abs(x)))
    assert np.all(np.abs(got - ref) <= bound), np.max(np.abs(got - ref) / bound)
    assert np.array_equal(_gmv(M, blk, x).view(np.int64), got.view(np.int64))          # run-to-run bits
    y0 = rng.standard_normal(n)
    assert np.array_equal(_gmv(M, blk, x, y0, accumulate=True), y0 + got)              # added exactly once


def test_empty_rows(M):
    import torch
    none = M.SubMatrix(buf=torch.zeros(0, dtype=torch.float64, device="cuda"), rows=0, cols=50, ld=50, is_transpose=True)
    y0 = np.arange(50.0)
    assert np.array_equal(_gmv(M, none, np.ones(50), y0), np.zeros(50))
    assert np.array_equal(_gmv(M, none, np.ones(50), y0, accumulate=True), y0)


def test_nan_and_inf_propagate(M):
    rng = np.random.default_rng(3)
    for n in (300, 6000):
        A = rng.standard_normal((200, n))
        A[3, 5] = np.nan
        A[7, 2] = np.inf
        A[11, :] = 0.0
        A[11, 4] = -np.inf
        x = rng.standard_normal(n)
        x[9] = np.inf
        with np.errstate(invalid="ignore", over="ignore"):
            t = np.sum(A * x, axis=1)
            ref = np.sum(A * t[:, None], axis=0)
        got = _gmv(M, _rowshard(M, A), x)
        assert np.array_equal(np.isnan(got), np.isnan(ref)) and np.array_equal(np.isposinf(got), np.isposinf(ref))
        assert np.array_equal(np.isneginf(got), np.isneginf(ref))


def test_two_launches_per_product(M):
    from marlin_b200 import _native as nat
    rt = M.Runtime.get()
    rng = np.random.default_rng(5)
    for m, n in [(1000, 64), (50, 9000)]:
        blk = _rowshard(M, rng.standard_normal((m, n)))
        x, y = _vec(M, rng.standard_normal(n)), _vec(M, np.zeros(n))
        rt.sync_stream()
        before = rt.lib.mb_launch_count(rt.ctx)
        nat.check(rt.lib.mb_block_gram_matvec(rt.ctx, blk.handle(), x.handle(), y.handle(), 0))
        assert rt.lib.mb_launch_count(rt.ctx) - before == 2


def test_argument_errors(M):
    from marlin_b200 import _native as nat
    rt = M.Runtime.get()
    blk = _rowshard(M, np.ones((4, 5)))
    v4, v5, w5, bf = _vec(M, np.ones(4)), _vec(M, np.ones(5)), _vec(M, np.ones(5)), blk.copy(nat.MB_BF16)
    assert rt.lib.mb_block_gram_matvec(rt.ctx, blk.handle(), v4.handle(), v5.handle(), 0) == nat.MB_ERR_DIM_MISMATCH
    assert rt.lib.mb_block_gram_matvec(rt.ctx, blk.handle(), v5.handle(), v4.handle(), 0) == nat.MB_ERR_DIM_MISMATCH
    assert rt.lib.mb_block_gram_matvec(rt.ctx, bf.handle(), v5.handle(), w5.handle(), 0) == nat.MB_ERR_UNSUPPORTED


# --------------------------------------------------------------------------------------------------- the solver
# The solver and computeSVD cases run in tests/eigs_gpu_worker.py, in a fresh process: their thousands of steps and operator
# calls leave nothing behind in this process, whose later tests inspect profiler traces.  The checks run here.
sys.path.insert(0, str(ROOT / "tests"))
import eigs_gpu_worker as W  # noqa: E402


@pytest.fixture(scope="module")
def one(tmp_path_factory):
    prefix = str(tmp_path_factory.mktemp("eigs") / "w")
    env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK")}
    env["EIGS_WORKER_OUT"] = prefix
    out = subprocess.run([sys.executable, str(ROOT / "tests" / "eigs_gpu_worker.py")], stdout=subprocess.PIPE,
                         stderr=subprocess.STDOUT, text=True, timeout=1500, env=env)
    assert out.returncode == 0 and "one eigs ok" in out.stdout, out.stdout[-6000:]
    return dict(np.load(prefix + ".one.npz"))


@pytest.mark.parametrize("kind,n,k", W.SOLVER_CASES)
def test_solver_through_the_c_abi(one, kind, n, k):
    import scipy.linalg
    G, lam = W.operator(kind, n, n + k)
    tol = 1e-10
    w, Z = one[f"solver.{kind}.{n}.{k}.w"], one[f"solver.{kind}.{n}.{k}.Z"]
    lmax = np.abs(lam).max()
    bound = tol * np.abs(w) + 1e-13 * lmax
    assert np.all(np.diff(w) <= 0)
    assert np.all(np.linalg.norm(G @ Z - Z * w, axis=0) <= bound)
    ref = scipy.linalg.eigh(G, eigvals_only=True)
    ref = ref[np.argsort(-np.abs(ref), kind="stable")][:k]
    assert np.all(np.abs(w - np.sort(ref)[::-1]) <= bound)
    assert np.abs(Z.T @ Z - np.eye(k)).max() <= 1e-12
    if k < n:
        d, _ = so.symmetric_eigs(lambda v: G @ v, n, k, tol, 300)
        assert np.all(np.abs(w - d) <= bound)


def test_solver_runs_out_of_restarts_with_the_reference_message(one):
    from marlin_b200 import _native as nat
    assert int(one["max_iter.code"]) == nat.MB_ERR_NO_CONVERGENCE
    assert str(one["max_iter.message"]) == ("ARPACK returns non-zero info = 1 Maximum number of iterations taken. "
                                            "(Refer ARPACK user guide for details)")


def test_solver_argument_errors(M):
    from marlin_b200 import _native as nat
    rt = M.Runtime.get()
    h = C.c_void_p()
    assert rt.lib.mb_eigs_create(rt.ctx, 10, 10, 10, 0.0, 5, 1, C.byref(h)) == nat.MB_ERR_INVALID_ARG
    assert rt.lib.mb_last_error() == b"Number of required eigenvalues 10 must be smaller than matrix dimension 10"
    assert rt.lib.mb_eigs_create(rt.ctx, 10, 3, 3, 0.0, 5, 1, C.byref(h)) == nat.MB_ERR_INVALID_ARG
    assert rt.lib.mb_eigs_create(rt.ctx, 10, 3, 6, 0.0, 0, 1, C.byref(h)) == nat.MB_ERR_INVALID_ARG
    assert not h.value


# --------------------------------------------------------------------------------------------------- computeSVD
@pytest.mark.parametrize("mode,k", W.TALL_CASES)
def test_compute_svd_tall(one, mode, k):
    A = W.tall()
    n = A.shape[1]
    s, V, Um = one[f"tall.{mode}.{k}.s"], one[f"tall.{mode}.{k}.V"], one[f"tall.{mode}.{k}.U"]
    ref = np.linalg.svd(A, compute_uv=False)
    assert len(s) == k and V.shape == (n, k)
    assert np.abs(s - ref[:k]).max() <= 1e-10 * ref[0]
    assert np.abs(V.T @ V - np.eye(k)).max() <= 1e-10
    assert np.abs(Um.T @ Um - np.eye(k)).max() <= 1e-10


def test_exact_rank_7_product_breaks_down(one):
    s, V = one["rank7.s"], one["rank7.V"]
    assert len(s) == 7 and V.shape == (40, 7)
    assert np.abs(s - np.linalg.svd(W.rank7(), compute_uv=False)[:7]).max() <= 1e-10 * s[0]


def test_wider_than_the_gramian_cap(one):
    A = W.wide()
    assert str(one["wide.capped"]) == "Argument with more than 65535 cols: 70000"
    s, V, Um, ref = one["wide.s"], one["wide.V"], one["wide.U"], one["wide.ref"]
    assert np.abs(s - ref[:5]).max() <= 1e-10 * ref[0]
    assert np.linalg.norm(A @ V - Um * s, axis=0).max() <= 1e-9 * ref[0]


@pytest.mark.parametrize("mode", W.KEEP_MODES)
def test_calls_without_the_keywords_keep_their_bits(one, mode):
    assert np.array_equal(one[f"keep.{mode}.s"], one["keep.ref.s"])
    assert np.array_equal(one[f"keep.{mode}.V"], one["keep.ref.V"])


def test_two_gloo_ranks_match_one(one, tmp_path):
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    env = dict(os.environ, EIGS_WORKER_OUT=str(tmp_path / "r"))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), str(ROOT / "tests" / "eigs_gpu_worker.py")]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900, env=env)
    assert out.returncode == 0, out.stdout[-4000:]
    for r in range(2):
        assert f"rank {r} eigs ok" in out.stdout
    s1, V1 = one["one.s"], one["one.V"]
    for layout in W.LAYOUTS:
        got = [np.load(str(tmp_path / f"r.{r}.{layout}.npz")) for r in range(2)]
        assert np.array_equal(got[0]["s"], got[1]["s"]) and np.array_equal(got[0]["V"], got[1]["V"]), layout
        assert np.abs(got[0]["s"] - s1).max() <= 1e-10 * s1[0], layout
        assert np.abs(np.abs(got[0]["V"].T @ V1) - np.eye(W.K)).max() <= 1e-8, layout

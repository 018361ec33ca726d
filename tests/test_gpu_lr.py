"""DenseVecMatrix.lr on the GPU: the fused gradient kernel (mb_lr_gradient), the on-device loop (mb_lr_train) and the
Python driver, against the step-by-step oracle (tests/lr_oracle.py) and float64 numpy / torch restatements."""
import ctypes as C
import os
import socket
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from tests import lr_oracle as lo

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
U = 2.0 ** -53


def _rowshard(A, ld=None, offset=0):
    """A row shard (transposed view, row r at offset + r * ld), as DenseVecMatrix holds its rows."""
    import torch
    import marlin_b200 as mb
    m, n = A.shape
    ld = ld or max(1, n)
    host = np.full(offset + m * ld + 1, np.nan)
    host[offset: offset + m * ld].reshape(m, ld)[:, :n] = A
    buf = torch.from_numpy(host).cuda()
    return mb.SubMatrix(buf=buf, rows=m, cols=n, ld=ld, offset=offset, is_transpose=True)


def _gradient(blk, w):
    import marlin_b200 as mb
    from marlin_b200 import _native as nat
    rt = mb.Runtime.get()
    rt.sync_stream()
    w = np.ascontiguousarray(w, dtype=np.float64)
    g = np.empty(blk.cols)
    nat.check(rt.lib.mb_lr_gradient(rt.ctx, blk.handle(), w.ctypes.data_as(nat.c_dp), g.ctypes.data_as(nat.c_dp)))
    return g


def _numpy_gradient(A, w):
    """float64 numpy: margins sequential in column order (elementwise IEEE ops, as ddot), numpy's exp, pairwise sums.
    Returns (gradient, bound) with bound = 2 (m + 2) u sum_r |x~_rj| (|g_r| + 1)."""
    m, n = A.shape
    X = A.copy()
    label = X[:, 0].copy()
    X[:, 0] = 1.0
    dot = np.zeros(m)
    for j in range(n):
        dot = dot + X[:, j] * w[j]
    with np.errstate(over="ignore"):
        g = 1.0 / (1.0 + np.exp(-1.0 * dot)) - label
    grad, bound = np.empty(n), np.empty(n)
    for c in range(0, n, 256):                                      # column chunks keep the temporaries small
        Xc = X[:, c:c + 256]
        grad[c:c + 256] = (Xc * g[:, None]).sum(axis=0)
        bound[c:c + 256] = 2.0 * (m + 2) * U * (np.abs(Xc) * (np.abs(g) + 1.0)[:, None]).sum(axis=0)
    return grad, bound


def _dyadic(m, n, seed):
    rng = np.random.default_rng(seed)
    A = rng.integers(-8, 9, (m, n)) / 4.0
    A[:, 0] = rng.integers(0, 2, m)
    return A


@pytest.mark.parametrize("m,n", [(1, 1), (8, 5), (64, 33), (1024, 129), (4096, 1025), (2048, 4097)])
def test_first_iteration_is_exact(m, n):
    """w = 0: gradientMul = 0.5 - label, dyadic features, m a power of two: every sum is exact, so lr(1, 1) is the oracle
    bit for bit."""
    import marlin_b200 as mb
    A = _dyadic(m, n, m + n)
    rows = [(i, A[i]) for i in range(m)]
    got = mb.DenseVecMatrix(rows).lr(1.0, 1)
    want = lo.lr(rows, 1.0, 1)
    assert got.shape == (n,)
    assert np.array_equal(got, want)


@pytest.mark.parametrize("m", [1, 7, 4099, 2 ** 17])
@pytest.mark.parametrize("n", [1, 2, 5, 31, 32, 33, 1023, 1024, 1025, 4097])
def test_gradient_at_arbitrary_w(m, n):
    """Against float64 numpy within the bound of _numpy_gradient: two orderings of the m-term sum plus a few ulps of g.
    The bound is too loose to see the margin's bits; test_margins_are_ddot_bit_for_bit pins those."""
    rng = np.random.default_rng(m * 31 + n)
    A = rng.standard_normal((m, n))
    A[:, 0] = rng.integers(0, 2, m)
    w = rng.standard_normal(n) / np.sqrt(n)
    got = _gradient(_rowshard(A), w)
    want, bound = _numpy_gradient(A, w)
    assert np.all(np.abs(got - want) <= bound), (m, n, np.max(np.abs(got - want) - bound))
    if m <= 7:
        assert np.all(np.abs(got - lo.gradient([(i, A[i]) for i in range(m)], w)) <= bound)


@pytest.mark.parametrize("n", [257, 1025])
def test_margins_are_ddot_bit_for_bit(n):
    """One row per call, label 0, margins near +700: g = 1 / (1 + exp(margin)) ~ 1e-305 changes by ~500 ulps per ulp of the
    margin (ulp(700) ~ 1.1e-13), while CUDA's and libm's exp differ by at most an ulp or two.  So a gradient within 4 ulps
    of the oracle's (mo_ddot_f2j margin, libm exp) means the device margin is the oracle's bit for bit.  The same rows
    with the margin summed in BLAS order instead (np.dot) miss that tolerance, so the check can tell them apart.  n = 257
    keeps the row resident in shared memory, n = 1025 streams it in pieces."""
    from oracle import reference_model as rm
    rng = np.random.default_rng(n)
    w = rng.standard_normal(n) / np.sqrt(n)
    w[0] = -700.0                                                          # the intercept weight carries the offset
    far = 0
    for r in range(16):
        x = rng.standard_normal(n)
        x[0] = 0.0                                                         # label 0
        got = _gradient(_rowshard(x.reshape(1, n)), w)
        xt = x.copy()
        xt[0] = 1.0
        want_g = lo.gradient_mul(rm.vector_dot(xt, w), 0.0)
        assert 1e-308 < want_g < 1e-290
        assert abs(got[0] - want_g) <= 4 * np.spacing(want_g), (r, (got[0] - want_g) / np.spacing(want_g))
        assert np.all(np.abs(got - xt * want_g) <= 4 * np.spacing(np.abs(xt * want_g)))
        far += abs(lo.gradient_mul(float(np.dot(xt, w)), 0.0) - want_g) > 4 * np.spacing(want_g)
    assert far >= 4, far


def test_views_misaligned_strided_and_column_major():
    """Rows at an odd ld starting 8 bytes past a 16-byte boundary, a wide ld, and a column-major block (staged) all give
    the bits of the packed row shard."""
    import marlin_b200 as mb
    rng = np.random.default_rng(5)
    A = rng.standard_normal((1000, 300))
    A[:, 0] = rng.integers(0, 2, 1000)
    w = rng.standard_normal(300) / 10
    ref = _gradient(_rowshard(A), w)
    for blk in (_rowshard(A, ld=301, offset=1), _rowshard(A, ld=1031, offset=3), mb.SubMatrix(A)):
        assert np.array_equal(_gradient(blk, w), ref)


def test_large_shard_against_torch():
    """1048576 x 1024 fp64 (8 GiB) against a float64 restatement on the device."""
    import torch
    import marlin_b200 as mb
    m, n = 1048576, 1024
    gen = torch.Generator(device="cuda").manual_seed(7)
    X = torch.randn(m, n, dtype=torch.float64, device="cuda", generator=gen)
    X[:, 0] = (torch.rand(m, device="cuda", generator=gen) < 0.5).double()
    w = torch.randn(n, dtype=torch.float64, device="cuda", generator=gen) / 32
    blk = mb.SubMatrix(buf=X.reshape(-1), rows=m, cols=n, ld=n, is_transpose=True)
    got = torch.from_numpy(_gradient(blk, w.cpu().numpy())).cuda()
    label = X[:, 0].clone()
    dot = X[:, 1:] @ w[1:] + w[0]
    g = 1.0 / (1.0 + torch.exp(-dot)) - label
    want = X.T @ g
    want[0] = g.sum()
    scale = X.abs().T @ (g.abs() + 1.0)
    scale[0] = (g.abs() + 1.0).sum()
    assert bool(((got - want).abs() <= 1e-9 * scale).all())
    del X, blk
    torch.cuda.empty_cache()


def test_fifty_iterations_against_oracle():
    """50 steps: exp (device vs libm) and the sum order differ in the last bits each step; relative 1e-10 of max |w|."""
    import marlin_b200 as mb
    rng = np.random.default_rng(50)
    A = rng.standard_normal((300, 17))
    A[:, 0] = rng.integers(0, 2, 300)
    rows = [(i, A[i]) for i in range(300)]
    got = mb.DenseVecMatrix(rows).lr(2.0, 50)
    want = lo.lr(rows, 2.0, 50)
    assert np.abs(got - want).max() <= 1e-10 * np.abs(want).max()


def test_margins_beyond_exp_range_and_nan():
    """|margin| > 710: exp overflows to Inf or underflows to 0, gradientMul is exactly -label or 1 - label.  A NaN feature
    makes its row's gradient NaN and so the whole sum."""
    A = np.array([[0.25, 1000.0], [0.75, -1000.0], [1.0, 800.0], [0.0, -720.0]])
    w = np.array([0.0, 1.0])
    got = _gradient(_rowshard(A), w)
    g = np.array([1 - 0.25, -0.75, 1 - 1.0, -0.0])
    want = np.array([g.sum(), (A[:, 1] * g).sum()])
    assert np.array_equal(got, want)
    B = A.copy()
    B[2, 1] = np.nan
    assert np.isnan(_gradient(_rowshard(B), w)).all()


def test_edges_iters_empty_dtype_gaps_input_and_repeatability():
    import torch
    import marlin_b200 as mb
    from marlin_b200 import _native as nat
    rng = np.random.default_rng(9)
    A = rng.standard_normal((4099, 33))
    A[:, 0] = rng.integers(0, 2, 4099)
    mat = mb.DenseVecMatrix([(i, A[i]) for i in range(4099)])
    assert np.array_equal(mat.lr(1.0, 0), np.zeros(33)) and np.array_equal(mat.lr(1.0, -3), np.zeros(33))
    before = mat.toBreeze().copy()
    w1, w2 = mat.lr(0.5, 7), mat.lr(0.5, 7)
    assert np.array_equal(w1, w2)                                        # bitwise reproducible
    assert np.array_equal(mat.toBreeze().view(np.int64), before.view(np.int64))    # the input is never written
    for empty in (mb.DenseVecMatrix([]), mb.DenseVecMatrix([], 0, 5), mb.DenseVecMatrix([], 4, 5)):
        with pytest.raises(nat.MarlinError) as e:
            empty.lr(1.0, 1)
        assert e.value.code == nat.MB_ERR_EMPTY
    bf = mb.SubMatrix(buf=torch.from_numpy(A.reshape(-1)).to(torch.bfloat16).cuda(), rows=4099, cols=33, ld=33,
                      is_transpose=True)
    with pytest.raises(nat.MarlinArgumentError) as e:
        mb.DenseVecMatrix(ids=np.arange(4099), data=bf, nRows=0, nCols=33).lr(1.0, 1)
    assert e.value.code == nat.MB_ERR_UNSUPPORTED
    with pytest.raises(nat.MarlinArgumentError) as e:
        _gradient(bf, np.zeros(33))
    assert e.value.code == nat.MB_ERR_UNSUPPORTED
    # rows of another width than numCols(): Breeze's dot would throw; no host buffer of the wrong size is handed out
    for n_cols in (3, 40):
        with pytest.raises(nat.MarlinArgumentError) as e:
            mb.DenseVecMatrix([(i, A[i]) for i in range(10)], 0, n_cols).lr(1.0, 1)
        assert e.value.code == nat.MB_ERR_DIM_MISMATCH
    # id gaps: dataSize = max id + 1 = 1000, not the 3 rows
    rows = [(999, A[0]), (0, A[1]), (500, A[2])]
    want = lo.lr(rows, 1.0, 3)
    assert np.abs(mb.DenseVecMatrix(rows).lr(1.0, 3) - want).max() <= 1e-12 * np.abs(want).max()


def test_two_ranks_agree_bitwise_and_match_one_rank(tmp_path):
    import marlin_b200 as mb
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    out_prefix = str(tmp_path / "w")
    env = dict(os.environ, LR_WORKER_OUT=out_prefix)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), str(ROOT / "tests" / "lr_gpu_worker.py")]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900, env=env)
    assert out.returncode == 0, out.stdout[-4000:]
    for r in range(2):
        assert f"rank {r} lr ok" in out.stdout
    rng = np.random.default_rng(21)
    A = rng.standard_normal((3000, 65))
    A[:, 0] = rng.integers(0, 2, A.shape[0])
    one = mb.DenseVecMatrix([(i, A[i]) for i in range(A.shape[0])]).lr(0.5, 20)
    for layout in ("interleaved", "one-rank-empty"):
        w = np.load(f"{out_prefix}.{layout}.0.npy")
        assert np.array_equal(w, np.load(f"{out_prefix}.{layout}.1.npy"))
        assert np.abs(w - one).max() <= 1e-12 * np.abs(one).max(), layout

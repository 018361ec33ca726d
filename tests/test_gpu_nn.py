"""The NeuralNetwork example on the GPU: mb_nn_gradient / mb_nn_step (the fused output-layer and backprop kernel between two
DMMA GEMMs, the hidden-weight gradient as K chunks of one grouped launch) and the Python driver, against the step-by-step
oracle (tests/nn_oracle.py)."""
import ctypes as C
import os
import socket
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from marlin_b200 import _native as nat
from tests import nn_oracle as no

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]


def _rel(got, want):
    return np.linalg.norm(got - want) / max(np.linalg.norm(want), 1e-300)


def _view(a, pad=0, offset=0):
    """A column-major block holding `a` with leading dimension rows + pad, `offset` elements into a NaN-filled buffer."""
    import torch
    import marlin_b200 as mb
    r, c = a.shape
    ld = max(1, r + pad)
    host = np.full(offset + ld * c + 1, np.nan)
    host[offset: offset + ld * c].reshape(c, ld)[:, :r] = a.T
    return mb.SubMatrix(buf=torch.from_numpy(host).cuda(), rows=r, cols=c, ld=ld, offset=offset)


class _Labels:
    def __init__(self, rt, ys):
        self.rt, self.ptrs = rt, []
        for y in ys:
            y = np.ascontiguousarray(y, np.int32)
            p = C.c_void_p()
            nat.check(rt.lib.mb_nn_labels_upload(rt.ctx, y.ctypes.data, len(y), C.byref(p)))
            self.ptrs.append(p)

    def array(self):
        return (C.c_void_p * len(self.ptrs))(*[p.value for p in self.ptrs])

    def free(self):
        for p in self.ptrs:
            self.rt.lib.mb_nn_labels_free(self.rt.ctx, p)


def _arr(blocks):
    return (nat.c_blk * len(blocks))(*[None if b is None else b.handle().value for b in blocks])


def _gradient(Xs, ys, W1, W2, scale, use_xt=True, d1_out=False, pad=0, offset=0):
    """(dW1, dW2, [D1_b] or None, launches) of one mb_nn_gradient call; every output starts as NaN."""
    import marlin_b200 as mb
    rt = mb.Runtime.get()
    H = W1.shape[1]
    xb = [_view(X, pad, offset) for X in Xs]
    xt = [_view(np.ascontiguousarray(X.T)) for X in Xs] if use_xt else None
    w1, w2 = _view(W1), _view(W2)
    g1, g2 = _view(np.full(W1.shape, np.nan)), _view(np.full(W2.shape, np.nan), pad=3)
    d1 = [_view(np.full((len(X), H), np.nan), pad=2 * pad) for X in Xs] if d1_out else None
    lab = _Labels(rt, ys)
    try:
        rt.sync_stream()
        before = rt.launch_count()
        nat.check(rt.lib.mb_nn_gradient(rt.ctx, _arr(xb), _arr(xt) if xt else None, lab.array(), len(Xs), w1.handle(), w2.handle(),
                                        scale, g1.handle(), g2.handle(), _arr(d1) if d1 else None))
        launches = rt.launch_count() - before
        rt.synchronize()
        return g1.toBreeze(), g2.toBreeze(), [d.toBreeze() for d in d1] if d1 else None, launches
    finally:
        lab.free()


def _case(rows, V, H, seed):
    rng = np.random.default_rng(seed)
    Xs = [rng.random((r, V)) * (rng.random((r, V)) < 0.25) for r in rows]
    ys = [rng.integers(0, 10, r) for r in rows]
    return Xs, ys, rng.normal(0, 0.2, (V, H)), rng.normal(0, 0.2, (H, 10))


def _check(Xs, ys, W1, W2, scale, got):
    dW1, dW2 = no.gradient(Xs, ys, W1, W2, scale)
    assert _rel(got[0], dW1) <= 1e-12 and _rel(got[1], dW2) <= 1e-12, (_rel(got[0], dW1), _rel(got[1], dW2))
    if got[2] is not None:
        for X, y, d in zip(Xs, ys, got[2]):
            assert _rel(d, no.backprop(X, y, W1, W2)[2]) <= 1e-12


@pytest.mark.parametrize("r", [1, 31, 32, 33, 1000, 1875])
def test_gradient_block_sizes(r):
    Xs, ys, W1, W2 = _case([r], 784, 100, r)
    got = _gradient(Xs, ys, W1, W2, 0.01, d1_out=r in (33, 1875))
    _check(Xs, ys, W1, W2, 0.01, got)


@pytest.mark.parametrize("H", [1, 10, 128, 129, 512, 1024])
def test_gradient_hidden_widths(H):
    """Both sides of the width up to which a row tile stays in shared memory (512)."""
    Xs, ys, W1, W2 = _case([700], 784, H, H)
    _check(Xs, ys, W1, W2, 0.5, _gradient(Xs, ys, W1, W2, 0.5, d1_out=H in (129, 1024)))


def test_chunked_and_transposed_a_paths_agree_and_are_the_ones_that_ran():
    """Three unequal blocks.  With XT the hidden-weight gradient is one grouped launch over K chunks: 3 GEMMs, 3 fused
    kernels, 1 grouped launch and 2 updates.  Without XT, and for an odd vectorLen (XT has an odd leading dimension), each
    block's product is a GEMM of its own: 3 + 3 + 3 + 2 launches."""
    Xs, ys, W1, W2 = _case([2100, 1030, 517], 784, 128, 7)
    a = _gradient(Xs, ys, W1, W2, 0.125)
    b = _gradient(Xs, ys, W1, W2, 0.125, use_xt=False)
    assert (a[3], b[3]) == (9, 11)
    _check(Xs, ys, W1, W2, 0.125, a)
    _check(Xs, ys, W1, W2, 0.125, b)
    assert _rel(a[0], b[0]) <= 1e-13 and np.array_equal(a[1], b[1])
    Xs, ys, W1, W2 = _case([1200, 600], 783, 64, 8)
    c = _gradient(Xs, ys, W1, W2, 0.125, d1_out=True)
    assert c[3] == 8
    _check(Xs, ys, W1, W2, 0.125, c)


def test_many_chunks_need_several_grouped_launches():
    """40 blocks of 600 rows: one chunk each, 32 entries in the first grouped launch and 8 in the second."""
    Xs, ys, W1, W2 = _case([600] * 40, 64, 16, 9)
    got = _gradient(Xs, ys, W1, W2, 1.0)
    assert got[3] == 40 + 40 + 2 + 2
    _check(Xs, ys, W1, W2, 1.0, got)


@pytest.mark.parametrize("pad,offset", [(1, 0), (4, 1), (7, 3)])
def test_strided_views(pad, offset):
    """X with ld > rows at an odd element offset (the GEMM's CUDA-core path), D1 written to a strided block."""
    Xs, ys, W1, W2 = _case([333, 64], 784, 96, pad)
    _check(Xs, ys, W1, W2, 0.25, _gradient(Xs, ys, W1, W2, 0.25, d1_out=True, pad=pad, offset=offset))


@pytest.mark.parametrize("H", [8, 640])
def test_exact_case(H):
    """Feature pairs that cancel against W1's row pairs give Z1 = 0, W2's row pairs cancel in Z2: every sigmoid is 0.5 and
    every product and sum is a small dyadic number, so the device result equals the oracle's exactly."""
    rng = np.random.default_rng(H)
    rows, V = [96, 40], 16
    Xs = []
    for r in rows:
        half = rng.integers(0, 5, (r, V // 2)).astype(np.float64)
        Xs.append(np.repeat(half, 2, axis=1))
    ys = [rng.integers(0, 10, r) for r in rows]
    w = rng.integers(-3, 4, (V // 2, H)).astype(np.float64)
    W1 = np.empty((V, H))
    W1[0::2], W1[1::2] = w, -w
    v = rng.integers(-4, 5, (H // 2, 10)).astype(np.float64)
    W2 = np.empty((H, 10))
    W2[0::2], W2[1::2] = v, -v
    got = _gradient(Xs, ys, W1, W2, 0.5, d1_out=True)
    dW1, dW2 = no.gradient(Xs, ys, W1, W2, 0.5)
    assert dW1.any() and dW2.any()
    assert np.array_equal(got[0], dW1) and np.array_equal(got[1], dW2)
    for X, y, d in zip(Xs, ys, got[2]):
        assert np.array_equal(d, no.backprop(X, y, W1, W2)[2])


def _synthetic(n=4096, V=784, seed=11):
    """Ten noisy class prototypes."""
    rng = np.random.default_rng(seed)
    proto = rng.random((10, V)) * (rng.random((10, V)) < 0.2)
    y = rng.integers(0, 10, n)
    return np.clip(proto[y] + 0.1 * rng.standard_normal((n, V)), 0.0, 1.0), y.astype(np.int32)


def _as_data(X, y, nblk):
    import marlin_b200 as mb
    from marlin_b200.matrix.block import BlockID
    bounds = no.rechunk(len(X), nblk)
    blocks = [(BlockID(b, 0), mb.SubMatrix(X[lo:hi])) for b, (lo, hi) in enumerate(bounds)]
    labels = {BlockID(b, 0): y[lo:hi] for b, (lo, hi) in enumerate(bounds)}
    return mb.BlockMatrix(blocks, len(X), X.shape[1], len(bounds), 1, sparse=False), labels, bounds


def _oracle_train(X, y, bounds, iterations, lr, executors, each, sel, H, seed):
    from marlin_b200.examples import neural_network as nn
    rng = np.random.default_rng(seed)
    W1, W2 = rng.normal(0.0, 0.2, (X.shape[1], H)), rng.normal(0.0, 0.2, (H, 10))
    batch = no.batch_size(sel, each, len(X))
    losses = []
    for _ in range(iterations):
        chosen = sorted(nn.genRandomBlocks(executors, each, sel, rng))
        W1, W2 = no.step([X[slice(*bounds[b])] for b in chosen], [y[slice(*bounds[b])] for b in chosen], W1, W2, lr, batch)
        losses.append(no.loss([X], [y], W1, W2))
    return W1, W2, losses


def test_train_matches_the_oracle_and_repeats_bit_for_bit():
    from marlin_b200.examples import neural_network as nn
    X, y = _synthetic()
    data, labels, bounds = _as_data(X, y, 8)
    args = (5, 2.0, 2, 4, 2, 64)
    W1, W2 = nn.train(data, labels, *args, seed=3)
    oW1, oW2, losses = _oracle_train(X, y, bounds, 5, 2.0, 2, 4, 2, 64, 3)
    assert _rel(W1, oW1) <= 1e-10 and _rel(W2, oW2) <= 1e-10
    assert all(b < a for a, b in zip(losses, losses[1:])), losses
    again = nn.train(data, labels, *args, seed=3)
    assert np.array_equal(again[0], W1) and np.array_equal(again[1], W2)
    # weights passed in, one more step from where the run stopped
    one = nn.train(data, labels, 1, 2.0, 2, 4, 4, 64, seed=0, hiddenWeight=W1, outputWeight=W2)
    want = no.step([X[slice(*b)] for b in bounds], [y[slice(*b)] for b in bounds], W1, W2, 2.0, len(X))
    assert _rel(one[0], want[0]) <= 1e-12 and _rel(one[1], want[1]) <= 1e-12


def test_two_ranks_match_one_rank(tmp_path):
    from marlin_b200.examples import neural_network as nn
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    prefix = str(tmp_path / "w")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), str(ROOT / "tests" / "nn_gpu_worker.py")]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900,
                         env=dict(os.environ, NN_WORKER_OUT=prefix))
    assert out.returncode == 0, out.stdout[-4000:]
    X, y = _synthetic(2048, 784, 5)
    data, labels, _ = _as_data(X, y, 8)
    W1, W2 = nn.train(data, labels, 3, 1.0, 2, 4, 2, 48, seed=4)
    for name, one in (("W1", W1), ("W2", W2)):
        a, b = (np.load(f"{prefix}.{name}.{r}.npy") for r in range(2))
        assert np.array_equal(a, b)
        assert _rel(a, one) <= 1e-12


def test_main_trains_on_a_libsvm_file(tmp_path):
    X, y = _synthetic(200, 784, 6)
    lines = [" ".join([str(l)] + [f"{j + 1}:{float(v)!r}" for j, v in enumerate(row) if v != 0.0]) for row, l in zip(X, y)]
    (tmp_path / "mnist").write_text("\n".join(lines) + "\n")
    out = subprocess.run([sys.executable, "-m", "marlin_b200.examples.neural_network", str(tmp_path / "mnist"), "2", "0.5", "2",
                          "2", "1", "20"], cwd=tmp_path, env=dict(os.environ, PYTHONPATH=str(ROOT)), stdout=subprocess.PIPE,
                         stderr=subprocess.STDOUT, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-3000:]
    W1 = np.loadtxt(tmp_path / "hiddenWeight", delimiter=",")
    W2 = np.loadtxt(tmp_path / "outputWeight", delimiter=",")
    assert W1.shape == (784, 20) and W2.shape == (20, 10) and np.isfinite(W1).all() and np.isfinite(W2).all()


def test_errors_take_no_memory_and_a_call_returns_what_it_took():
    import torch
    import marlin_b200 as mb
    from tests.test_gpu_temporaries import _Pool
    rt = mb.Runtime.get()
    lib, ctx = rt.lib, rt.ctx
    Xs, ys, W1, W2 = _case([100], 784, 32, 1)
    x, w1, w2, g1, g2 = _view(Xs[0]), _view(W1), _view(W2), _view(W1 * 0), _view(W2 * 0)
    p = C.c_void_p(0x5E47)
    bad = np.array([0, 10, 3], np.int32)
    assert lib.mb_nn_labels_upload(ctx, bad.ctypes.data, 3, C.byref(p)) == nat.MB_ERR_INVALID_ARG and p.value is None
    assert b"label 10 of row 1" in lib.mb_last_error()
    lab = _Labels(rt, ys)
    pool = _Pool()
    rt.sync_stream()

    def call(x=x, w1=w1, w2=w2, g1=g1):
        return lib.mb_nn_gradient(ctx, _arr([x]), None, lab.array(), 1, w1.handle(), w2.handle(), 1.0, g1.handle(), g2.handle(), None)

    try:
        assert call() == nat.MB_OK
        rt.synchronize()
        before = pool.used()
        bf16 = mb.SubMatrix(buf=torch.zeros(100 * 784, dtype=torch.bfloat16, device="cuda"), rows=100, cols=784, ld=100)
        assert call(x=bf16) == nat.MB_ERR_UNSUPPORTED
        assert call(w2=_view(np.zeros((33, 10)))) == nat.MB_ERR_DIM_MISMATCH                # H mismatch
        assert call(w1=_view(np.zeros((783, 32))), g1=_view(np.zeros((783, 32)))) == nat.MB_ERR_DIM_MISMATCH
        assert call(g1=_view(np.zeros((784, 31)))) == nat.MB_ERR_DIM_MISMATCH
        assert lib.mb_nn_step(ctx, _arr([x]), None, lab.array(), 0, w1.handle(), w2.handle(), 1.0) == nat.MB_ERR_INVALID_ARG
        rt.synchronize()
        assert pool.used() == before
        pool.reset_high()
        assert call() == nat.MB_OK
        rt.synchronize()
        assert pool.high() > before and pool.used() == before
    finally:
        lab.free()

"""The sharded dist-mode LU / Cholesky / inverse and the grouped Schur update under it.

mb_block_schur_update must give every C[e] the bits of mb_block_gemm(A, B) -> tmp; mb_block_sub(C, tmp), on every path
(grouped launches, transposed B, odd leading dimensions, views, vector shapes), with the DMMA reference instances on and
off.  One rank of the sharded factorizations must give the bits of the per-block call sequence they replace, restated
here from public SubMatrix calls; more ranks are checked by tests/factor_dist_gpu_worker.py."""
import ctypes as C
import os
import socket
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]
G2_MAX_ENTRIES, G2_MAX_OPS = 64, 32


@pytest.fixture(scope="module")
def mb():
    import marlin_b200 as mb
    mb.Runtime.get()
    yield mb
    # the factorizations above leave a few GB in torch's cache: hand it back so later modules start as they would alone
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _rt(mb):
    rt = mb.Runtime.get()
    rt.sync_stream()
    return rt


def _launches(mb):
    rt = mb.Runtime.get()
    torch.cuda.synchronize()
    return int(rt.lib.mb_launch_count(rt.ctx))


def _schur(mb, entries):
    from marlin_b200.matrix.factorizations import schur_update
    schur_update(entries)


def _reference(mb, c, a, b):
    """C - A B the way the per-block path computes it."""
    return c.subtract(a.multiply(b))


def _block(mb, a, ld=None, offset=0):
    """A device block holding a (column-major), optionally with a larger leading dimension and an element offset."""
    m, n = a.shape
    ld = ld or max(1, m)
    buf = np.zeros(offset + ld * n)
    for j in range(n):
        buf[offset + j * ld: offset + j * ld + m] = a[:, j]
    return mb.SubMatrix(buf=torch.from_numpy(buf).cuda(), rows=m, cols=n, ld=ld, offset=offset)


def _bits(x):
    return x.toBreeze().view(np.uint64)


CASES = [(1, 1, 1), (1, 7, 5), (7, 1, 5), (6, 5, 1), (37, 37, 37), (38, 38, 38), (1000, 1000, 1000), (1001, 1001, 1001),
         (128, 256, 384), (256, 128, 128), (300, 200, 130)]


@pytest.mark.parametrize("reference_mma", [0, 1])
def test_schur_update_is_gemm_then_sub_bitwise(mb, reference_mma):
    rt = mb.Runtime.get()
    rng = np.random.default_rng(5 + reference_mma)
    nat = mb._native
    nat.check(rt.lib.mb_set_dmma_reference(rt.ctx, reference_mma))
    try:
        entries, want = [], []
        for (m, n, k) in CASES:
            c, a, b = rng.standard_normal((m, n)), rng.standard_normal((m, k)), rng.standard_normal((k, n))
            cb, ab, bb = _block(mb, c), _block(mb, a), _block(mb, b)
            want.append(_bits(_reference(mb, cb, ab, bb)))
            entries.append((cb, ab, bb))
        # odd leading dimension, a sliced view, a transposed B (Cholesky's L_ci^T), an odd element offset
        c, a, b = rng.standard_normal((200, 150)), rng.standard_normal((200, 96)), rng.standard_normal((150, 96))
        cb, ab, bt = _block(mb, c, ld=201), _block(mb, a, ld=203), _block(mb, b).t
        want.append(_bits(_reference(mb, cb, ab, bt))); entries.append((cb, ab, bt))
        big = _block(mb, rng.standard_normal((400, 400)))
        cv = big.slice(128, 384, 0, 256)
        av, bv = _block(mb, rng.standard_normal((300, 300))).slice(0, 256, 128, 256), _block(mb, rng.standard_normal((128, 256)))
        want.append(_bits(_reference(mb, cv, av, bv))); entries.append((cv, av, bv))
        bt2 = _block(mb, rng.standard_normal((256, 256))).t
        c2, a2 = _block(mb, rng.standard_normal((256, 256))), _block(mb, rng.standard_normal((256, 256)))
        want.append(_bits(_reference(mb, c2, a2, bt2))); entries.append((c2, a2, bt2))
        c3, a3, b3 = _block(mb, rng.standard_normal((64, 64)), offset=1), _block(mb, rng.standard_normal((64, 64)), offset=1), \
            _block(mb, rng.standard_normal((64, 64)), offset=1)
        want.append(_bits(_reference(mb, c3, a3, b3))); entries.append((c3, a3, b3))
        _schur(mb, entries)
        for (cb, _, _), w in zip(entries, want):
            assert np.array_equal(_bits(cb), w), cb.rows
    finally:
        nat.check(rt.lib.mb_set_dmma_reference(rt.ctx, 0))


def test_schur_update_exact_on_small_integers(mb):
    rng = np.random.default_rng(11)
    entries, want = [], []
    for (m, n, k) in [(1000, 1000, 1000), (37, 38, 129), (256, 256, 1)]:
        c, a, b = (rng.integers(-8, 9, s).astype(np.float64) for s in ((m, n), (m, k), (k, n)))
        entries.append((_block(mb, c), _block(mb, a), _block(mb, b)))
        want.append(c - a @ b)
    _schur(mb, entries)
    for (cb, _, _), w in zip(entries, want):
        assert np.array_equal(cb.toBreeze(), w)


def _packing_model(entries):
    """Launches of the grouped path: entries in order, a launch closed when the next entry would exceed
    G2_MAX_ENTRIES or bring a 33rd distinct A or B operand."""
    launches, ne, a_ops, b_ops = 0, 0, set(), set()
    for (_, a, b) in entries:
        if ne == G2_MAX_ENTRIES or (a not in a_ops and len(a_ops) == G2_MAX_OPS) or (b not in b_ops and len(b_ops) == G2_MAX_OPS):
            launches += 1
            ne, a_ops, b_ops = 0, set(), set()
        ne += 1
        a_ops.add(a); b_ops.add(b)
    return launches + (1 if ne else 0)


@pytest.mark.parametrize("rows,cols", [(9, 9), (40, 2), (2, 40), (33, 33)])
def test_schur_update_packing_and_launch_count(mb, rows, cols):
    """A trailing update over a rows x cols block grid with shared row (X_r) and column (Y_c) operands."""
    rng = np.random.default_rng(rows * 100 + cols)
    s = 128
    X = [_block(mb, rng.integers(-4, 5, (s, s)).astype(np.float64)) for _ in range(rows)]
    Y = [_block(mb, rng.integers(-4, 5, (s, s)).astype(np.float64)) for _ in range(cols)]
    Cs = {(r, c): _block(mb, rng.integers(-4, 5, (s, s)).astype(np.float64)) for r in range(rows) for c in range(cols)}
    want = {k: v.toBreeze() - X[k[0]].toBreeze() @ Y[k[1]].toBreeze() for k, v in Cs.items()}
    entries = [(Cs[(r, c)], X[r], Y[c]) for r in range(rows) for c in range(cols)]
    before = _launches(mb)
    _schur(mb, entries)
    got = _launches(mb) - before
    assert got == _packing_model([(None, id(a), id(b)) for (_, a, b) in entries])
    for k, v in Cs.items():
        assert np.array_equal(v.toBreeze(), want[k])
    before = _launches(mb)
    _schur(mb, [])
    rt = _rt(mb)
    mb._native.check(rt.lib.mb_block_schur_update(rt.ctx, 0, None, None, None))
    assert _launches(mb) == before


def test_schur_update_errors(mb):
    rt = _rt(mb)
    nat = mb._native
    rng = np.random.default_rng(3)
    a, b, c = (_block(mb, rng.standard_normal((64, 64))) for _ in range(3))

    def call(entries):
        n = len(entries)
        arr = lambda j: (nat.c_blk * n)(*[e[j].handle() for e in entries])
        return rt.lib.mb_block_schur_update(rt.ctx, n, arr(0), arr(1), arr(2))

    assert call([(c, a, _block(mb, rng.standard_normal((63, 64))))]) == nat.MB_ERR_DIM_MISMATCH
    assert call([(_block(mb, rng.standard_normal((64, 63))), a, b)]) == nat.MB_ERR_DIM_MISMATCH
    assert call([(c, c, b)]) == nat.MB_ERR_INVALID_ARG
    assert call([(c, a, c.t)]) == nat.MB_ERR_INVALID_ARG
    assert call([(c, a, b), (c.slice(0, 32, 0, 32), a.slice(0, 32, 0, 64), b.slice(0, 64, 0, 32))]) == nat.MB_ERR_INVALID_ARG
    assert call([(c, a, b), (b.slice(0, 64, 0, 32), a, a.slice(0, 64, 0, 32))]) == nat.MB_ERR_INVALID_ARG
    assert rt.lib.mb_block_schur_update(rt.ctx, -1, None, None, None) == nat.MB_ERR_INVALID_ARG


# ------------------------------------------------------------------------------------- one rank and several ranks
# The factorizations run in tests/factor_dist_gpu_worker.py, each rank count in fresh processes, so the thousands of
# block calls of the one-rank chains leave nothing behind in this process.
def _run_worker(tmp_path, ranks, chain=False):
    """The worker on `ranks` gloo ranks: ({rank: what it saved}, its output)."""
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    prefix = str(tmp_path / f"w{ranks}")
    env = dict(os.environ, FACTOR_WORKER_OUT=prefix, FACTOR_WORKER_CHAIN="1" if chain else "0")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={ranks}", "--master-addr",
           "127.0.0.1", "--master-port", str(port), str(ROOT / "tests" / "factor_dist_gpu_worker.py")]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800, env=env)
    assert out.returncode == 0, out.stdout[-6000:]
    for r in range(ranks):
        assert f"rank {r} factor ok" in out.stdout, out.stdout[-6000:]
    return {r: dict(np.load(f"{prefix}.{r}.npz")) for r in range(ranks)}, out.stdout


@pytest.fixture(scope="module")
def one_rank(tmp_path_factory):
    return _run_worker(tmp_path_factory.mktemp("one"), 1, chain=True)


def test_one_rank_matches_the_per_block_chain(one_rank):
    """(n, base) in (10, 3) (last block 1 x 1), (301, 40) and (3001, 200) (more than 64 updates per step): L/U, pivots
    (also with keepUnfactoredDiagonal), the Cholesky factor and the inverse equal the per-block call sequence bit for bit."""
    _, stdout = one_rank
    for n, base in ((10, 3), (301, 40), (3001, 200)):
        assert f"chain {n} {base} ok" in stdout, stdout[-6000:]


def test_two_and_three_ranks_match_one_rank(tmp_path, one_rank):
    one = one_rank[0][0]
    assert one["chol_error"][0] != 0
    for ranks in (2, 3):
        for r, got in _run_worker(tmp_path, ranks)[0].items():
            for key in one:
                if key == "peak_3001":
                    continue
                assert np.array_equal(got[key].view(np.uint64), one[key].view(np.uint64)), (ranks, r, key)
            if ranks == 2:
                assert got["peak_3001"][0] <= 0.7 * one["peak_3001"][0], (got["peak_3001"], one["peak_3001"])


def test_matrix_lu_decompose_example(tmp_path, mb):
    import scipy.linalg as sla
    from marlin_b200.examples import matrix_lu_decompose
    src = ROOT / "tests" / "golden" / "a.100.100"
    out = tmp_path / "lu"
    matrix_lu_decompose.main([str(src), "100", "100", str(out), "1"])
    A = mb.MTUtils.loadMatrixFile(None, str(src)).toBreeze()
    LU = mb.MTUtils.loadMatrixFile(None, str(out)).toBreeze()
    P, L, U = sla.lu(A)
    assert np.abs(LU - (np.tril(L, -1) + U)).max() <= 1e-10 * max(1.0, np.abs(U).max())
    L2, U2 = np.tril(LU, -1) + np.eye(100), np.triu(LU)
    _, perm = mb.MTUtils.loadMatrixFile(None, str(src)).luDecompose()
    assert np.abs(A[perm] - L2 @ U2).max() <= 1e-10 * np.abs(A).max()
    with pytest.raises(SystemExit) as e:
        matrix_lu_decompose.main([str(src), "100"])
    assert e.value.code == -1

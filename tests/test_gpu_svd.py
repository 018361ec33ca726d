"""DenseVecMatrix.computeSVD on the GPU: the split-K DMMA Gramian, the Jacobi eigensolver and the Python driver, against
host fp64 arithmetic, numpy / LAPACK and the step-by-step oracle (tests/svd_oracle.py)."""
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
SUITE_ROWS = [(0, [2.0, 0.0, 8.0, 6.0, 0.0]), (1, [1.0, 6.0, 0.0, 1.0, 7.0]), (2, [5.0, 0.0, 7.0, 4.0, 0.0]),
              (3, [7.0, 0.0, 8.0, 5.0, 0.0]), (4, [0.0, 10.0, 0.0, 0.0, 7.0])]


def _rowshard(A):
    import torch
    import marlin_b200 as mb
    m, n = A.shape
    buf = torch.from_numpy(np.ascontiguousarray(A).reshape(-1)).cuda()
    return mb.SubMatrix(buf=buf, rows=m, cols=n, ld=max(1, n), is_transpose=True)


@pytest.mark.parametrize("m", [1, 7, 4096, 2 ** 17])
@pytest.mark.parametrize("n", [1, 2, 5, 127, 128, 129, 1024])
def test_gramian(m, n):
    import marlin_b200 as mb
    rng = np.random.default_rng(m * 7919 + n)
    A = rng.standard_normal((m, n))
    ref = A.T @ A
    scale = np.abs(A).T @ np.abs(A)
    for blk in (_rowshard(A), mb.SubMatrix(A)):
        G1 = blk.gramian().toBreeze()
        G2 = blk.gramian().toBreeze()
        assert np.array_equal(G1, G1.T), (m, n, blk)
        assert np.array_equal(G1, G2), (m, n, blk)
        assert (np.abs(G1 - ref) / np.maximum(scale, 1e-300)).max() <= 1e-10, (m, n, blk)


def _inputs(n, rng):
    A = rng.standard_normal((n + 7, n))
    S = rng.standard_normal((n, n))
    yield "psd", A.T @ A
    yield "indefinite", S + S.T
    yield "diagonal", np.diag(rng.standard_normal(n))
    yield "zero", np.zeros((n, n))
    yield "identity", np.eye(n)


@pytest.mark.parametrize("n", [1, 2, 3, 5, 64, 255, 256, 1000])
def test_symmetric_eigen_against_lapack(n):
    import marlin_b200 as mb
    rng = np.random.default_rng(n)
    for kind, G in _inputs(n, rng):
        blk = mb.SubMatrix(G)
        w, V = blk.symmetricEigen()
        w2, V2 = blk.symmetricEigen()
        V, V2 = V.toBreeze(), V2.toBreeze()
        assert np.array_equal(w, w2) and np.array_equal(V, V2), kind
        wr, Vr = np.linalg.eigh(G)
        order = sorted(range(n), key=lambda i: (-abs(wr[i]), i))
        wr, Vr = wr[order], Vr[:, order]
        assert np.all(np.abs(w[:-1]) >= np.abs(w[1:])), kind
        norm2 = max(np.abs(wr).max(), 1e-300)
        assert np.abs(w - wr).max() <= 1e-12 * norm2, (kind, np.abs(w - wr).max() / norm2)
        assert np.abs(V.T @ V - np.eye(n)).max() <= 1e-12, kind
        assert np.linalg.norm(G @ V - V * w) <= 1e-12 * max(np.linalg.norm(G), 1e-300), kind
        if kind in ("psd", "indefinite"):
            gaps = np.abs(np.diff(wr))
            sep = np.ones(n, dtype=bool)
            if n > 1:
                sep[:-1] &= gaps > 1e-3 * norm2
                sep[1:] &= gaps > 1e-3 * norm2
            for j in np.flatnonzero(sep):
                d = min(np.abs(V[:, j] - Vr[:, j]).max(), np.abs(V[:, j] + Vr[:, j]).max())
                assert d <= 1e-10, (kind, j, d)


def test_suite_case():
    import marlin_b200 as mb
    mat = mb.DenseVecMatrix(SUITE_ROWS)
    U, s, V = mat.computeSVD(3, True)
    assert np.array_equal(np.round(s, 2), [17.92, 15.17, 3.56])
    A = np.array([r for _, r in SUITE_ROWS])
    assert np.abs(U.toBreeze() - A @ V / s).max() <= 1e-12


@pytest.fixture(scope="module")
def tall():
    rng = np.random.default_rng(20000)
    return rng.standard_normal((20000, 300))


@pytest.mark.parametrize("k", [10, 150, 300])
@pytest.mark.parametrize("mode", ["auto", "local-svd", "local-eigs", "dist-eigs"])
def test_compute_svd_tall(tall, k, mode):
    import marlin_b200 as mb
    A = tall
    n = A.shape[1]
    try:
        so.svd_mode(n, k, mode)
    except ValueError:
        pytest.skip(f"the reference's requires reject k={k} in {mode} mode")
    mat = mb.DenseVecMatrix(list(enumerate(A)))
    U, s, V = mat.computeSVD(k, computeU=True, mode=mode)
    ref = np.linalg.svd(A, compute_uv=False)
    assert len(s) == k and V.shape == (n, k)
    assert np.abs(s - ref[:k]).max() <= 1e-10 * ref[0]
    _, so_s, _ = so.compute_svd(list(enumerate(A)), n, k, mode=mode)
    assert np.abs(s - so_s).max() <= 1e-10 * ref[0]
    Um = U.toBreeze()
    assert np.abs(V.T @ V - np.eye(k)).max() <= 1e-10
    assert np.abs(Um.T @ Um - np.eye(k)).max() <= 1e-10
    if k == n:
        assert np.linalg.norm(A - (Um * s) @ V.T) <= 1e-10 * np.linalg.norm(A)


def test_effective_rank_of_an_exact_rank_7_product():
    import marlin_b200 as mb
    rng = np.random.default_rng(7)
    A = rng.integers(-9, 10, (400, 7)).astype(np.float64) @ rng.integers(-9, 10, (7, 40)).astype(np.float64)
    _, s, V = mb.DenseVecMatrix(list(enumerate(A))).computeSVD(20, rCond=1e-6)
    assert len(s) == 7 and V.shape == (40, 7)
    assert np.abs(s - np.linalg.svd(A, compute_uv=False)[:7]).max() <= 1e-10 * s[0]


def test_reference_errors():
    import marlin_b200 as mb
    mat = mb.DenseVecMatrix(SUITE_ROWS)
    for args, msg in [((0,), "Request up to n singular values but got k=0 and n=5."),
                      ((6,), "Request up to n singular values but got k=6 and n=5."),
                      ((2, False, 1e-9, "lanczos"), "Do not support mode lanczos."),
                      ((5, False, 1e-9, "local-eigs"), "k must be smaller than n in local-eigs mode but got k=5 and n=5."),
                      ((5, False, 1e-9, "dist-eigs"), "k must be smaller than n in dist-eigs mode but got k=5 and n=5.")]:
        with pytest.raises(mb.MarlinArgumentError) as ei:
            mat.computeSVD(*args)
        assert str(ei.value) == msg


def test_quarter_of_config_4():
    """262144 x 1024 from MTUtils.randomDenVecMatrix: A v_i = s_i u_i and orthonormal factors."""
    import torch
    import marlin_b200 as mb
    mat = mb.MTUtils.randomDenVecMatrix(None, 262144, 1024, seed=4)
    U, s, V = mat.computeSVD(10, computeU=True)
    assert len(s) == 10 and np.all(np.diff(s) <= 0)
    Um = U.toBreeze()
    Av = mat.multiply(V).toBreeze()
    assert np.abs(Av - Um * s).max() <= 1e-9 * s[0]
    assert np.abs(V.T @ V - np.eye(10)).max() <= 1e-10
    assert np.abs(Um.T @ Um - np.eye(10)).max() <= 1e-9
    del U, mat
    torch.cuda.empty_cache()


def test_two_ranks_agree_bitwise():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), str(ROOT / "tests" / "svd_gpu_worker.py")]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900, env=dict(os.environ))
    assert out.returncode == 0, out.stdout[-4000:]
    for r in range(2):
        assert f"rank {r} svd ok" in out.stdout


@pytest.mark.parametrize("n", [3000, 3001])
def test_gramian_large_n_in_place(n):
    """Past two waves of triangle tiles K is not split: no workspace, the product is written into G and mirrored in place
    (odd n: the row shard takes the CUDA-core path, the column-major block the DMMA path)."""
    import marlin_b200 as mb
    from marlin_b200 import _native as nat
    m = 4096
    rt = mb.Runtime.get()
    assert rt.lib.mb_gramian_workspace_bytes(n, m, torch_sm_count()) == 0
    rng = np.random.default_rng(n)
    A = rng.standard_normal((m, n))
    ref = A.T @ A
    scale = np.abs(A).T @ np.abs(A)
    for blk in (_rowshard(A), mb.SubMatrix(A)):
        G1 = blk.gramian().toBreeze()
        assert np.array_equal(G1, G1.T) and np.array_equal(G1, blk.gramian().toBreeze())
        assert (np.abs(G1 - ref) / scale).max() <= 1e-10
    assert nat.MB_OK == 0


def torch_sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count

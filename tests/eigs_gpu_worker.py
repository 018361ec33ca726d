"""Worker for computeSVD's Lanczos path (tests/test_gpu_eigs.py), so that the many solver steps and operator calls run in a
fresh process and leave nothing behind in the pytest process, whose later tests inspect profiler traces.

    python tests/eigs_gpu_worker.py              one process: every solver and computeSVD case, saved to $EIGS_WORKER_OUT.one.npz
    torch.distributed.run ... eigs_gpu_worker.py two gloo ranks (both may share one GPU): uneven row splits and a rank
                                                 that holds no rows; each rank saves its s and V and checks that the rows
                                                 of U stay with the rows of A it holds
"""
import ctypes as C
import os
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import marlin_b200 as mb
from marlin_b200 import _native as nat

K = 10
LAYOUTS = ("uneven", "rank-0-empty")
SOLVER_CASES = [(kind, n, k) for n, k in [(120, 5), (40, 39)]
                for kind in ("separated", "clustered", "repeated", "rank-deficient")
                if not (kind == "repeated" and k < n - 1)]     # one Krylov sequence holds one vector of a repeated eigenspace
TALL_CASES = [(mode, k) for mode in ("dist-eigs", "local-eigs", "auto") for k in (10, 150)]
KEEP_MODES = ("auto", "local-eigs", "dist-eigs", "local-svd")


def matrix():
    return np.random.default_rng(4242).standard_normal((6000, 200))


def tall():
    return np.random.default_rng(20000).standard_normal((20000, 300))


def rank7():
    rng = np.random.default_rng(7)
    return rng.integers(-9, 10, (400, 7)).astype(np.float64) @ rng.integers(-9, 10, (7, 40)).astype(np.float64)


def wide():
    rng = np.random.default_rng(70000)
    return rng.standard_normal((2000, 70000)) / (1.0 + np.arange(2000.0))[:, None]


def spectrum(kind, n, rng):
    if kind == "separated":
        return np.linspace(1.0, 100.0, n)[::-1] * (1 + 0.1 * rng.random(n))
    if kind == "clustered":                    # the four largest 1e-8 apart, relative
        lam = np.linspace(0.1, 50.0, n)
        lam[-4:] = 100.0 * (1 + 1e-8 * np.arange(4))
        return lam
    if kind == "repeated":
        lam = np.linspace(1.0, 60.0, n)
        lam[-4:] = 80.0
        lam[:5] = 0.5
        return lam
    lam = np.linspace(1.0, 30.0, n)            # exactly rank-deficient: a third of the spectrum is zero
    lam[: n // 3] = 0.0
    return lam


def operator(kind, n, seed):
    """(G = Q diag(lam) Q^T, lam) for a solver case."""
    rng = np.random.default_rng(seed)
    lam = spectrum(kind, n, rng)
    Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    G = (Q * lam) @ Q.T
    return (G + G.T) / 2, lam


def eigs(G, k, ncv, tol, max_iter):
    """The C ABI loop with Op = G (mb_block_gemv); -> (w, Z)."""
    rt = mb.Runtime.get()
    rt.sync_stream()
    n = G.shape[0]
    g = mb.SubMatrix(G)
    h = C.c_void_p()
    nat.check(rt.lib.mb_eigs_create(rt.ctx, n, k, ncv, tol, max_iter, 1557, C.byref(h)))
    try:
        ido, x, y = C.c_int32(0), nat.c_blk(), nat.c_blk()
        while True:
            nat.check(rt.lib.mb_eigs_step(rt.ctx, h, C.byref(ido), C.byref(x), C.byref(y)))
            if ido.value == 99:
                break
            nat.check(rt.lib.mb_block_gemv(rt.ctx, g.handle(), x, y, 0))
        w = np.zeros(k)
        Z = mb.SubMatrix.empty(n, k)
        nconv, iters = C.c_int32(), C.c_int32()
        nat.check(rt.lib.mb_eigs_result(rt.ctx, h, w.ctypes.data_as(nat.c_dp), Z.handle(), C.byref(nconv), C.byref(iters)))
        assert nconv.value >= k
        return w, Z.toBreeze()
    finally:
        rt.lib.mb_eigs_destroy(h)


def run_one(out):
    import torch
    mb.Runtime.get()
    res = {}
    for kind, n, k in SOLVER_CASES:
        G, _ = operator(kind, n, n + k)
        res[f"solver.{kind}.{n}.{k}.w"], res[f"solver.{kind}.{n}.{k}.Z"] = eigs(G, k, min(2 * k, n), 1e-10, 300)
    G, _ = operator("clustered", 400, 9)
    try:
        eigs(G, 3, 6, 1e-14, 1)
        res["max_iter.code"], res["max_iter.message"] = np.array(0), np.array("")
    except nat.MarlinError as e:
        res["max_iter.code"], res["max_iter.message"] = np.array(e.code), np.array(e.message)
    A = tall()
    mat = mb.DenseVecMatrix(list(enumerate(A)))
    for mode, k in TALL_CASES:
        U, s, V = mat.computeSVD(k, computeU=True, mode=mode, tol=1e-10)
        res[f"tall.{mode}.{k}.s"], res[f"tall.{mode}.{k}.V"], res[f"tall.{mode}.{k}.U"] = s, V, U.toBreeze()
    _, res["rank7.s"], res["rank7.V"] = mb.DenseVecMatrix(list(enumerate(rank7()))).computeSVD(
        20, rCond=1e-6, mode="dist-eigs", tol=1e-10)
    # calls without the keywords, beside the existing path restated: Gramian, Jacobi, rank, V
    small = mb.DenseVecMatrix(list(enumerate(A[:4000, :120])))
    w, vblk = small.data.gramian().symmetricEigen()
    sig = np.sqrt(np.abs(w))
    sk = nat.load().mb_svd_rank(sig.ctypes.data_as(nat.c_dp), len(sig), 10, 1e-9)
    res["keep.ref.s"], res["keep.ref.V"] = sig[:sk], vblk.slice(0, 120, 0, sk).toBreeze()
    for mode in KEEP_MODES:
        _, res[f"keep.{mode}.s"], res[f"keep.{mode}.V"] = small.computeSVD(10, True, 1e-9, mode)
    _, res["one.s"], res["one.V"] = mb.DenseVecMatrix(list(enumerate(matrix()))).computeSVD(K, mode="dist-eigs", tol=1e-10)
    del mat, small
    W = wide()
    At = torch.from_numpy(W).cuda()
    shard = mb.SubMatrix(buf=At.reshape(-1), rows=W.shape[0], cols=W.shape[1], ld=W.shape[1], is_transpose=True)
    wm = mb.DenseVecMatrix(ids=np.arange(W.shape[0]), data=shard, nRows=W.shape[0], nCols=W.shape[1])
    try:
        wm.computeSVD(5, mode="dist-eigs")
        res["wide.capped"] = np.array("")
    except mb.MarlinArgumentError as e:
        res["wide.capped"] = np.array(str(e))
    U, res["wide.s"], res["wide.V"] = wm.computeSVD(5, computeU=True, mode="dist-eigs", tol=1e-10)
    res["wide.U"] = U.toBreeze()
    # the singular values from the eigenvalues of A A^T (2000 x 2000, formed on the device): accurate to eps s_0 at the top
    res["wide.ref"] = np.sqrt(np.abs(np.linalg.eigvalsh((At @ At.T).cpu().numpy())))[::-1]
    np.savez(out + ".one.npz", **res)
    print("one eigs ok", flush=True)


def run_ranks(out):
    import torch.distributed as dist
    dist.init_process_group("gloo")
    rank = dist.get_rank()
    mb.Runtime.get()
    A = matrix()
    for layout in LAYOUTS:
        if layout == "uneven":
            ids = range(0, 1700) if rank == 0 else range(1700, A.shape[0])
        else:
            ids = range(A.shape[0]) if rank == 1 else range(0)
        rows = [(i, A[i]) for i in ids]
        mat = mb.DenseVecMatrix(rows, A.shape[0], A.shape[1])
        U, s, V = mat.computeSVD(K, computeU=True, mode="dist-eigs", tol=1e-10)
        np.savez(out + f".{rank}.{layout}.npz", s=s, V=V)
        assert set(int(i) for i in U.ids) == set(ids), layout
        if len(U.ids):
            mine = U.data.toBreeze()
            want = A[U.ids] @ V / s
            assert np.abs(mine - want).max() <= 1e-10 * np.abs(want).max(), layout
    dist.barrier()
    dist.destroy_process_group()
    print(f"rank {rank} eigs ok")


if __name__ == "__main__":
    if "RANK" in os.environ:
        run_ranks(os.environ["EIGS_WORKER_OUT"])
    else:
        run_one(os.environ["EIGS_WORKER_OUT"])

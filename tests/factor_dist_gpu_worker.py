"""Worker for the sharded dist-mode LU / Cholesky / inverse (gloo for the gathers and exchanges, so the ranks may share
one GPU).  Rows are dealt to the ranks by row id; every rank checks that it holds exactly the result blocks elem_owner
gives it and that DenseVecMatrix.toBreeze is never called, then saves what it collected (and its peak device memory)
for the caller to compare across ranks and with the same worker run on one rank."""
import os
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import marlin_b200 as mb
from marlin_b200 import comm


def matrices(n):
    """A general matrix and a symmetric positive definite one.  The latter is a product of small integers, so it is exact
    and the same in every process whatever BLAS threading numpy uses there."""
    rng = np.random.default_rng(n)
    A = rng.standard_normal((n, n)) + n ** 0.5 * np.eye(n)
    B = rng.integers(-3, 4, (n, n)).astype(np.float64)
    return A, B @ B.T + n * np.eye(n)


def rows(a):
    rank, ws = mb.runtime.world()
    return mb.DenseVecMatrix([(i, a[i]) for i in range(a.shape[0]) if i % ws == rank], a.shape[0], a.shape[1])


def _no_gather(self):
    raise AssertionError("dist mode gathered the matrix")


def _held(bm, nb):
    rank, ws = mb.runtime.world()
    got = sorted((b.row, b.column) for b, _ in bm.blocks)
    return got, [k for k in got if comm.elem_owner(k[0], k[1], nb, ws) != rank]


def run():
    from marlin_b200.matrix import factorizations as fz
    from marlin_b200.matrix.dense_vec_matrix import DenseVecMatrix
    rank, ws = mb.runtime.world()
    out = {}
    saved = DenseVecMatrix.toBreeze
    for n, base in ((301, 40), (6001, None)):
        A, S = matrices(n)
        mats = (rows(A), rows(S))
        DenseVecMatrix.toBreeze = _no_gather
        try:
            if base is None:
                res = {"lu": mats[0].luDecompose()}
                nb = fz.grid(n, 1000)[0]
            else:
                res = {"lu": mats[0].luDecompose("dist", base), "lu_keep": mats[0].luDecompose("dist", base, True),
                       "chol": mats[1].choleskyDecompose("dist", base), "inv": mats[0].inverse("dist", base)}
                nb = fz.grid(n, base)[0]
        finally:
            DenseVecMatrix.toBreeze = saved
        for name, r in res.items():
            bm, perm = r if isinstance(r, tuple) else (r, None)
            held, foreign = _held(bm, nb)
            assert not foreign, (name, foreign)
            if perm is not None:
                out[f"{name}_{n}_perm"] = np.asarray(perm)
            out[f"{name}_{n}"] = bm.toBreeze()
    # peak device memory of a sharded LU beyond what the caller held at entry
    A, _ = matrices(3001)
    M = rows(A)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    entry = torch.cuda.memory_allocated()
    lu, _ = M.luDecompose("dist", 200)
    torch.cuda.synchronize()
    out["peak_3001"] = np.array([torch.cuda.max_memory_allocated() - entry])
    del lu
    # a failing diagonal block: the same error on every rank, and the run goes on
    n = 90
    code = 0
    try:
        rows(-np.eye(n) - np.ones((n, n))).choleskyDecompose("dist", 30)
    except (mb.MarlinError, mb.MarlinArgumentError) as e:
        code = e.code
    out["chol_error"] = np.array([code])
    return out


# ---- the per-block call sequence of the one-rank algorithms
def _perm_matrix(perm):
    pm = np.zeros((len(perm), len(perm)))
    pm[np.arange(len(perm)), np.asarray(perm)] = 1.0
    return mb.SubMatrix(pm, device=torch.device("cuda"))


def _chain_lu(blocks, nb, sub, n, keep):
    cur, p_array, done = dict(blocks), [0] * n, {}
    for i in range(nb):
        first = cur[(i, i)]
        packed, perm = first.lu()
        for j, pj in enumerate(perm):
            p_array[i * sub + j] = i * sub + int(pj)
        if i == nb - 1:
            done[(i, i)] = packed
            break
        pm = _perm_matrix(perm)
        done[(i, i)] = first if keep else packed
        u = {k: packed.solveTriangular(pm.multiply(v), lower=True, unit=True) for k, v in cur.items() if k[0] == i and k[1] > i}
        l = {k: packed.t.solveTriangular(v.t, lower=True, unit=False).transpose() for k, v in cur.items() if k[0] > i and k[1] == i}
        done.update(u); done.update(l)
        cur = {(r, c): v.subtract(l[(r, i)].multiply(u[(i, c)])) for (r, c), v in cur.items() if r > i and c > i}
    out = {}
    for (r, c), blk in done.items():
        if r > c:
            arr = p_array[sub * r: (n if r == nb - 1 else sub * r + sub)]
            blk = _perm_matrix([a - sub * r for a in arr]).multiply(blk)
        out[(r, c)] = blk
    return out, p_array


def _chain_cholesky(blocks, nb):
    cur, done = {k: v for k, v in blocks.items() if k[0] >= k[1]}, {}
    for i in range(nb):
        l = cur[(i, i)].cholesky()
        done[(i, i)] = l
        if i == nb - 1:
            break
        col = {k: l.solveTriangular(v.t, lower=True, unit=False).transpose() for k, v in cur.items() if k[0] > i and k[1] == i}
        done.update(col)
        cur = {(r, c): v.subtract(col[(r, i)].multiply(col[(c, i)].t)) for (r, c), v in cur.items() if c > i and r >= c}
    return done


def _chain_inverse(blocks, nb):
    cur, sc = dict(blocks), {}
    for i in range(nb):
        if i == nb - 1:
            cur = {k: v.inverse() for k, v in cur.items()}
            break
        second = {k: v for k, v in cur.items() if k[0] == i and k[1] > i}
        third = {k: v for k, v in cur.items() if k[0] > i and k[1] == i}
        inv = cur[(i, i)].inverse()
        sc[(i, 0)] = inv
        sc[(i, 1)] = {k: inv.multiply(v).multiply(-1.0) for k, v in second.items()}
        sc[(i, 2)] = {k: v.multiply(inv).multiply(-1.0) for k, v in third.items()}
        cur = {(r, c): v.subtract(third[(r, i)].multiply(inv).multiply(second[(i, c)]))
               for (r, c), v in cur.items() if r > i and c > i}
    for i in range(nb - 2, -1, -1):
        s2, s3, rng = sc[(i, 1)], sc[(i, 2)], range(i + 1, nb)

        def total(pairs):
            acc = None
            for a, b in pairs:
                acc = a.multiply(b) if acc is None else a.multiply(b, out=acc, accumulate=True)
            return acc

        mt = {(r, i): total((cur[(r, c)], s3[(c, i)]) for c in rng) for r in rng}
        ms = {(i, c): total((s2[(i, r)], cur[(r, c)]) for r in rng) for c in rng}
        first = total((s2[(i, c)], mt[(c, i)]) for c in rng).add(sc[(i, 0)])
        cur.update(ms); cur.update(mt)
        cur[(i, i)] = first
    return cur


def _grid(A, base):
    from marlin_b200.matrix.factorizations import grid
    n = A.shape[0]
    nb, sub = grid(n, base)
    return {(r, c): mb.SubMatrix(A[r * sub:min(n, (r + 1) * sub), c * sub:min(n, (c + 1) * sub)], device=torch.device("cuda"))
            for r in range(nb) for c in range(nb)}, nb, sub


def _collected(bm):
    return {(b.row, b.column): s.toBreeze() for b, s in bm.blocks}


def _same(got, want):
    assert sorted(got) == sorted(want)
    for k in want:
        w = want[k].toBreeze() if not isinstance(want[k], np.ndarray) else want[k]
        assert np.array_equal(got[k].view(np.uint64), w.view(np.uint64)), k


def chain_check():
    """One rank: each result equals bit for bit the per-block call sequence the sharded algorithms replace, restated
    here from public SubMatrix calls."""
    for n, base in ((10, 3), (301, 40), (3001, 200)):
        A, S = matrices(n)
        M = mb.DenseVecMatrix([(i, A[i]) for i in range(n)], n, n)
        blocks, nb, sub = _grid(A, base)
        for keep in (False, True):
            lu, perm = M.luDecompose("dist", base, keepUnfactoredDiagonal=keep)
            want, wperm = _chain_lu(blocks, nb, sub, n, keep)
            assert perm == wperm
            _same(_collected(lu), want)
        chol = mb.DenseVecMatrix([(i, S[i]) for i in range(n)], n, n).choleskyDecompose("dist", base)
        _same(_collected(chol), _chain_cholesky(_grid(S, base)[0], nb))
        _same(_collected(M.inverse("dist", base)), _chain_inverse(blocks, nb))
        print(f"chain {n} {base} ok", flush=True)


def main():
    import torch.distributed as dist
    dist.init_process_group("gloo")
    rank = dist.get_rank()
    mb.Runtime.get()
    if os.environ.get("FACTOR_WORKER_CHAIN") == "1" and dist.get_world_size() == 1:
        chain_check()
    out = run()
    codes = [None] * dist.get_world_size()
    dist.all_gather_object(codes, int(out["chol_error"][0]))
    assert codes[0] != 0 and len(set(codes)) == 1, codes
    np.savez(os.environ["FACTOR_WORKER_OUT"] + f".{rank}.npz", **out)
    dist.barrier()
    dist.destroy_process_group()
    print(f"rank {rank} factor ok")


if __name__ == "__main__":
    main()

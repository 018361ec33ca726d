"""Two-rank worker for the DistributedMatrix API (gloo for the gathers and exchanges, so both ranks may share one GPU):
the rows are dealt to the ranks by row id, every method runs, and rank 0 saves what it collected for the caller to
compare with one rank.  `run` is also what the caller runs on one rank."""
import os
import sys
from pathlib import Path

import numpy as np
import torch.distributed as dist

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import marlin_b200 as mb


def _ints(m, n, seed):
    return np.random.default_rng(seed).integers(-8, 9, size=(m, n)).astype(np.float64)


def run(M):
    rank, ws = M.runtime.world()

    def rows(a, ids=None):
        ids = range(a.shape[0]) if ids is None else ids
        return M.DenseVecMatrix([(int(i), a[int(i)]) for i in ids if int(i) % ws == rank], a.shape[0], a.shape[1])

    a, b, c = _ints(13, 7, 1), _ints(13, 5, 2), _ints(13, 4, 3)
    wide = _ints(9, 6, 4)
    x = rows(a)
    out = {
        "slice_row": x.sliceByRow(2, 9).toBreeze(),
        "slice_col": x.sliceByColumn(1, 5).toBreeze(),
        "sub": x.getSubMatrix(3, 12, 0, 3).toBreeze(),
        "cbind_dense": x.cBind(rows(b, ids=[0, 1, 2, 4, 6, 7, 8, 10, 12])).toBreeze(),
        "cbind_block_relabel": rows(wide).toBlockMatrix(3, 2).cBind(rows(wide).toBlockMatrix(3, 2)).toBreeze(),
        "cbind_block_rows": rows(a).toBlockMatrix(2, 2).cBind(rows(c).toBlockMatrix(2, 2)).toBreeze(),
        "repeat_row_dense": M.MTUtils.repeatByRow(x, 3).toBreeze(),
        "repeat_col_dense": M.MTUtils.repeatByColumn(x, 2).toBreeze(),
        "repeat_row_block": M.MTUtils.repeatByRow(rows(wide).toBlockMatrix(3, 2), 2).toBreeze(),
        "repeat_col_block": M.MTUtils.repeatByColumn(rows(a).toBlockMatrix(2, 2), 3).toBreeze(),
        "element_multiply": rows(a).toBlockMatrix(3, 2).elementMultiply(rows(_ints(13, 7, 5)).toBlockMatrix(3, 2)).toBreeze(),
        # the relabelled blocks keep their ranks, which differ from a fresh 3 x 4 grid's: add moves blocks between ranks
        "add_moved": rows(wide).toBlockMatrix(3, 2).cBind(rows(wide).toBlockMatrix(3, 2))
                     .add(rows(np.hstack([wide, wide]) * 2.0).toBlockMatrix(3, 4)).toBreeze(),
        "zeros": M.MTUtils.zerosDenVecMatrix(None, 10, 3).toBreeze(),
        "ones": M.MTUtils.onesDenVecMatrix(None, 10, 3).toBreeze(),
    }
    big = _ints(5000, 37, 6)
    rnd = np.random.default_rng(7).standard_normal((3000, 41))
    for name, mat in (("int", rows(big)), ("rand", rows(rnd))):
        for mode in ("1", "inf", "fro"):
            if name == "rand" and mode != "inf":
                continue                                   # "1" and "fro" are exact on integers only
            out[f"norm_{mode}_{name}"] = np.float64(mat.norm(mode))
    # a shard the kernel rejects on rank 0 only: every rank raises the same error
    bad = rows(big)
    if rank == 0:
        bad = M.DenseVecMatrix(ids=bad.ids, data=bad.data.copy(M._native.MB_BF16), nRows=bad.numRows(), nCols=bad.numCols())
    try:
        bad.norm("inf")
        raise AssertionError("no error")
    except M.MarlinArgumentError as e:
        assert e.code == M._native.MB_ERR_UNSUPPORTED and str(e) == "mb_block_norm: fp64 blocks only", str(e)
    return out


def main():
    dist.init_process_group("gloo")
    rank = dist.get_rank()
    mb.Runtime.get()
    out = run(mb)
    if rank == 0:
        np.savez(os.environ["DMS_API_WORKER_OUT"] + f".{rank}.npz", **out)
    dist.barrier()
    dist.destroy_process_group()
    print(f"rank {rank} dms api ok")


if __name__ == "__main__":
    main()

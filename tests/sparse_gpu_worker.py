"""Two-rank worker (NCCL, one process per GPU) for BlockMatrix.multiply with sparse blocks: sparse tiles cross ranks as
packed buffers next to dense tiles, every rank agrees that a matrix has sparse blocks, and each C block equals the host
restatement of the reference loops (tests/sparse_oracle.py), P0 + P1 in kk order, bit for bit."""
import os
import sys
from pathlib import Path

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import marlin_b200 as mb

from tests import sparse_oracle as so


def gather_tiles(bm):
    """Every tile of `bm` on every rank: ("s", csc tuple) or ("d", ndarray)."""
    mine = []
    for b, s in bm.blocks:
        if s.isSparse:
            cp, ri, va = s.sparseBlock.to_host()
            mine.append(((b.row, b.column), ("s", (s.rows, s.cols, cp, ri, va))))
        else:
            mine.append(((b.row, b.column), ("d", s.toBreeze())))
    out = [None] * dist.get_world_size()
    dist.all_gather_object(out, mine)
    return dict(x for part in out for x in part)


def main():
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    rank, ws = dist.get_rank(), dist.get_world_size()
    mb.Runtime.get()
    M, K, N = 301, 257, 199
    As = mb.MTUtils.randomBlockMatrix(None, M, K, 2, 2, (True, 0.05), seed=31)
    Bs = mb.MTUtils.randomBlockMatrix(None, K, N, 2, 2, (True, 0.05), seed=32)
    Ad = mb.MTUtils.randomBlockMatrix(None, M, K, 2, 2, seed=33)
    Bd = mb.MTUtils.randomBlockMatrix(None, K, N, 2, 2, seed=34)
    # a user-built matrix whose only sparse block lives on rank 0: the flag is still the same on both ranks
    user = mb.BlockMatrix([(b, s) for b, s in As.blocks if rank == 0 or not s.isSparse], M, K, 2, 2)
    assert user._has_sparse() and As._has_sparse() and not Ad._has_sparse()
    for name, A, B in (("ss", As, Bs), ("ds", Ad, Bs), ("sd", As, Bd)):
        C = A.multiply(B)
        ta, tb = gather_tiles(A), gather_tiles(B)
        prod = {"ss": so.spgemm, "ds": so.mult_dense_sparse, "sd": so.mult_sparse_dense}[name]
        for b, blk in C.blocks:
            ref = prod(ta[(b.row, 0)][1], tb[(0, b.column)][1]) + prod(ta[(b.row, 1)][1], tb[(1, b.column)][1])
            got = blk.toBreeze()
            assert got.shape == ref.shape and np.array_equal(got.view(np.int64), ref.view(np.int64)), (name, b.row, b.column)
        dense = A.toDenseBlocks().multiply(B.toDenseBlocks()).toBreeze()
        full = C.toBreeze()
        assert np.abs(full - dense).max() <= 1e-10 * max(1.0, np.abs(dense).max()), name
    dist.barrier()
    dist.destroy_process_group()
    print(f"rank {rank} sparse ok")


if __name__ == "__main__":
    main()

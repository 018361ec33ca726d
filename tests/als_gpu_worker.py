"""Two-rank worker for CoordinateMatrix.ALS (gloo for the exchange of factor rows, so both ranks may share one GPU): the
entries are dealt to the ranks interleaved; every rank returns the rows of its own blocks.  Each rank saves (ids, factors)
for the caller to compare with the one-rank result bit for bit."""
import os
import sys
from pathlib import Path

import numpy as np
import torch.distributed as dist

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import marlin_b200 as mb


def data():
    rng = np.random.default_rng(5)
    nnz = 6000
    rows = rng.integers(0, 300, nnz)
    cols = rng.integers(0, 200, nnz)
    vals = rng.uniform(-2, 5, nnz).astype(np.float32)
    return rows, cols, vals


def main():
    dist.init_process_group("gloo")
    rank, ws = dist.get_rank(), dist.get_world_size()
    mb.Runtime.get()
    rows, cols, vals = data()
    mine = np.arange(len(rows)) % ws == rank
    m = mb.CoordinateMatrix((rows[mine], cols[mine], vals[mine]))
    for implicit in (False, True):
        U, P = m.ALS(12, 2, 0.05, 5, 3, implicit, 0.7, seed=99)
        out = os.environ["ALS_WORKER_OUT"] + f".{int(implicit)}.{rank}.npz"
        np.savez(out, uid=U.ids, U=U.data.toBreeze() if len(U.ids) else np.zeros((0, 12)), pid=P.ids,
                 P=P.data.toBreeze() if len(P.ids) else np.zeros((0, 12)))
    # lambda = 0: product 0 is rated 0.0 by users 11, 13, 15, 17 only, so its factor solves to exactly zero and those users'
    # normal equations are exactly zero.  They are all in user block 1, solved on rank 1 alone; both ranks must raise
    # the same error instead of one rank waiting in the exchange.
    sr, sc, sv = [], [], []
    for u in range(40):
        if u in (11, 13, 15, 17):
            sr.append(u); sc.append(0); sv.append(0.0)
        else:
            for k in (u % 29, (u + 7) % 29, (u + 13) % 29, (u + 19) % 29):
                sr.append(u); sc.append(k + 1); sv.append(1.0 + (u * 7 + k) % 5)
    sr, sc, sv = np.array(sr), np.array(sc), np.array(sv, np.float32)
    mine = np.arange(len(sr)) % ws == rank
    try:
        mb.CoordinateMatrix((sr[mine], sc[mine], sv[mine])).ALS(2, 1, 0.0, 2, 2, seed=3)
        raise AssertionError("no error")
    except mb.MarlinError as e:
        assert "entity 11 are not positive definite" in str(e), str(e)
    print(f"rank {rank} singular raised")
    # a duplicate (row, col) held by one rank only fails toDenseVecMatrix on every rank
    dup = [((rank, 1), 1.0)] + ([((5, 2), 2.0), ((5, 2), 3.0)] if rank == 1 else [])
    try:
        mb.CoordinateMatrix(dup).toDenseVecMatrix()
        raise AssertionError("no error")
    except mb.MarlinArgumentError as e:
        assert "Found duplicate indices: 2." in str(e), str(e)
    print(f"rank {rank} duplicate raised")
    dist.barrier()
    dist.destroy_process_group()
    print(f"rank {rank} als ok")


if __name__ == "__main__":
    main()

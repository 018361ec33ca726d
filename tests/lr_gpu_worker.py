"""Two-rank worker for DenseVecMatrix.lr (gloo for the exchange of the partial gradients, so both ranks may share one GPU):
interleaved row ids, and one rank without rows.  w must be bitwise equal across ranks; each rank saves it for the caller
to compare with the one-rank result."""
import os
import sys
from pathlib import Path

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import marlin_b200 as mb


def main():
    dist.init_process_group("gloo")
    rank, ws = dist.get_rank(), dist.get_world_size()
    mb.Runtime.get()
    rng = np.random.default_rng(21)
    A = rng.standard_normal((3000, 65))
    A[:, 0] = rng.integers(0, 2, A.shape[0])
    for layout in ("interleaved", "one-rank-empty"):
        if layout == "interleaved":
            rows = [(i, A[i]) for i in range(A.shape[0]) if i % ws == rank]
        else:
            rows = [(i, A[i]) for i in range(A.shape[0])] if rank == 1 else []
        mat = mb.DenseVecMatrix(rows, 0, A.shape[1])
        w = mat.lr(0.5, 20)
        got = [None] * ws
        dist.all_gather_object(got, w)
        for w2 in got:
            assert np.array_equal(w2, w), layout
        print(f"rank {rank} {layout} w = {w[:3]}")
        np.save(os.environ["LR_WORKER_OUT"] + f".{layout}.{rank}.npy", w)
    dist.barrier()
    dist.destroy_process_group()
    print(f"rank {rank} lr ok")


if __name__ == "__main__":
    main()

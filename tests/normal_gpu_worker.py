"""Two-rank worker for the StandardNormalGenerator generators (gloo for the gathers, so both ranks may share one GPU):
each generator deals its partitions to the ranks, and rank 0 saves what it collected for the caller to compare with one
rank.  `run` is also what the caller runs on one rank."""
import os
import sys
from pathlib import Path

import numpy as np
import torch.distributed as dist

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import marlin_b200 as mb
from marlin_b200.utils.mt_utils import OnesGenerator, StandardNormalGenerator


def run(M):
    g = StandardNormalGenerator(-1.5, 2.25)
    sp = M.MTUtils.randomSpaVecMatrix(None, 57, 40, 0.2, numPartitions=5, distribution=g, seed=23)
    vec = M.MTUtils.randomDistVector(None, 101, 4, distribution=g, seed=24)
    return {
        **{f"vector_{i}": piece.toBreeze() for i, piece in vec.vectors},       # this rank's pieces
        "dense": M.MTUtils.randomDenVecMatrix(None, 61, 29, numPartitions=5, distribution=g, seed=21).toBreeze(),
        "block": M.MTUtils.randomBlockMatrix(None, 50, 37, 3, 4, distribution=g, seed=22).toBreeze(),
        "spvec": sp.toBreeze(),
        "ones": M.MTUtils.randomBlockMatrix(None, 9, 7, 2, 2, distribution=OnesGenerator(), seed=25).toBreeze(),
    }


def main():
    dist.init_process_group("gloo")
    rank = dist.get_rank()
    mb.Runtime.get()
    out = run(mb)
    if rank == 0:
        np.savez(os.environ["NORMAL_WORKER_OUT"] + f".{rank}.npz", **out)
    dist.barrier()
    dist.destroy_process_group()
    print(f"rank {rank} normal generators ok")


if __name__ == "__main__":
    main()

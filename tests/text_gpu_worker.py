"""Two-rank worker for the matrix-file writer (gloo, so both ranks may share one GPU): each rank saves its own rows of one
DenseVecMatrix to TEXT_WORKER_OUT, which gives one part file per rank."""
import os
import sys
from pathlib import Path

import numpy as np
import torch.distributed as dist

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import marlin_b200 as mb


def rows(rank):
    """Rank r holds rows 50 r .. 50 r + 49 of a 100 x 23 matrix."""
    rng = np.random.default_rng(31 + rank)
    return [(50 * rank + i, rng.standard_normal(23) * 10.0 ** (i % 9 - 4)) for i in range(50)]


def main():
    dist.init_process_group("gloo")
    rank = dist.get_rank()
    mb.Runtime.get()
    mb.DenseVecMatrix(rows(rank), nRows=100, nCols=23).saveWithDescription(os.environ["TEXT_WORKER_OUT"])
    dist.barrier()
    dist.destroy_process_group()
    print(f"rank {rank} text ok")


if __name__ == "__main__":
    main()

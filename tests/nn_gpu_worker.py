"""Two-rank worker for the NeuralNetwork example (gloo for the exchange of the gradient sums, so both ranks may share one
GPU): each rank holds one executor's four blocks.  The weights must be bitwise equal across ranks; each rank saves them for
the caller to compare with the one-rank result."""
import os
import sys
from pathlib import Path

import numpy as np
import torch.distributed as dist

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import marlin_b200 as mb
from marlin_b200.examples import neural_network as nn
from marlin_b200.matrix.block import BlockID
from tests.nn_oracle import rechunk
from tests.test_gpu_nn import _synthetic


def main():
    dist.init_process_group("gloo")
    rank, ws = dist.get_rank(), dist.get_world_size()
    mb.Runtime.get()
    X, y = _synthetic(2048, 784, 5)
    bounds = rechunk(len(X), 8)
    mine = [b for b in range(8) if b * ws // 8 == rank]
    data = mb.BlockMatrix([(BlockID(b, 0), mb.SubMatrix(X[slice(*bounds[b])])) for b in mine], len(X), 784, 8, 1, sparse=False)
    labels = {BlockID(b, 0): y[slice(*bounds[b])] for b in mine}
    W1, W2 = nn.train(data, labels, 3, 1.0, 2, 4, 2, 48, seed=4)
    for name, W in (("W1", W1), ("W2", W2)):
        got = [None] * ws
        dist.all_gather_object(got, W)
        assert all(np.array_equal(g, W) for g in got), name
        np.save(os.environ["NN_WORKER_OUT"] + f".{name}.{rank}.npy", W)
    dist.barrier()
    dist.destroy_process_group()
    print(f"rank {rank} nn ok")


if __name__ == "__main__":
    main()

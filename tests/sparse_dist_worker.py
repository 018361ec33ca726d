"""Worker for the two-rank gloo test of sparse tiles (CPU): a sparse tile travels through comm.exchange as one packed
buffer whose size both ranks agree on before allocating, and "this matrix has sparse blocks" is the same on every rank,
even one that holds no sparse block."""
import sys
from pathlib import Path

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import marlin_b200 as mb
from marlin_b200 import comm
from marlin_b200.matrix.sparse_matrix import SparseBlock

from tests import sparse_oracle as so


def main():
    dist.init_process_group("gloo")
    rank, ws = dist.get_rank(), dist.get_world_size()
    assert ws == 2
    cpu = torch.device("cpu")
    rng = np.random.default_rng(0)                       # same on both ranks
    tiles = {key: so.random_csc(rng, 13 + key, 9 + 2 * key, 0.3, empty_cols=0.2) for key in range(4)}
    tiles[3] = so.random_csc(rng, 5, 4, 0.0)             # an empty tile travels too
    mine = {key: SparseBlock.from_host(*t, device=cpu) for key, t in tiles.items() if key % 2 == rank}
    # nnz is agreed before any rank allocates (BlockMatrix._multiply_same_grid gathers it the same way)
    bm = mb.BlockMatrix([])
    nnz = dict(bm._all_gather_meta([(key, b.nnz) for key, b in mine.items()]))
    assert nnz == {key: t[3].size for key, t in tiles.items()}
    sends = [(key % 2, 1 - key % 2, key) for key in range(4)]
    got = comm.exchange(sends, {key: b.pack() for key, b in mine.items()},
                        lambda key: torch.empty(SparseBlock.packed_bytes(tiles[key][1], nnz[key]), dtype=torch.uint8), rank)
    assert sorted(got) == [key for key in range(4) if key % 2 != rank]
    for key, buf in got.items():
        blk = SparseBlock.unpack(buf, tiles[key][0], tiles[key][1], nnz[key])
        for x, y in zip(blk.to_host(), tiles[key][2:]):
            assert np.array_equal(x, y)
    # the sparse flag is global: rank 1 holds only a dense block here
    blocks = [(mb.BlockID(0, 0), mb.SubMatrix(sparse=mine[0]))] if rank == 0 else \
        [(mb.BlockID(0, 1), mb.SubMatrix(np.ones((3, 3)), device=cpu))]
    assert mb.BlockMatrix(blocks)._has_sparse()
    dense = [(mb.BlockID(0, rank), mb.SubMatrix(np.ones((3, 3)), device=cpu))]
    assert not mb.BlockMatrix(dense)._has_sparse()
    dist.barrier()
    dist.destroy_process_group()
    print(f"rank {rank} ok")


if __name__ == "__main__":
    main()

"""Two-rank worker for the PageRank example (gloo for the gathers and the exchange, so both ranks may share one GPU): the
link pairs are dealt to the ranks by source page, each rank builds the in-links of the piece it owns, and the pieces are
exchanged every iteration.  Each rank saves the pieces it holds for the caller to compare with one rank bit for bit."""
import os
import sys
from pathlib import Path

import numpy as np
import torch.distributed as dist

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import marlin_b200 as mb
from marlin_b200.examples import page_rank as pr
from tests import pagerank_oracle as po

N, ITERATIONS = 3001, 6


def data():
    return po.random_graph(N, seed=77)


def main():
    dist.init_process_group("gloo")
    rank, ws = dist.get_rank(), dist.get_world_size()
    mb.Runtime.get()
    src, dst = data()
    keep = src % ws == rank
    ids, rowptr, cols, vals = po.link_rows(src[keep], dst[keep], N)
    links = mb.SparseVecMatrix((ids, rowptr, cols, vals), N, N)
    ranks = pr.pageRank(links, ITERATIONS)
    out = {f"p{i}": v.toBreeze().reshape(-1) for i, v in ranks.vectors}
    np.savez(os.environ["PAGERANK_WORKER_OUT"] + f".{rank}.npz", **out)
    try:
        pr.pageRank(mb.SparseVecMatrix((np.zeros(0, np.int64), np.zeros(1, np.int64), np.zeros(0, np.int64), np.zeros(0)),
                                       3, 3), 1)
        raise AssertionError("no error")
    except mb.MarlinArgumentError as e:
        assert "not supported matrix or vector" in str(e), str(e)
    print(f"rank {rank} small graph raised")
    dist.barrier()
    dist.destroy_process_group()
    print(f"rank {rank} pagerank ok")


if __name__ == "__main__":
    main()

"""Two-rank worker for SparseVecMatrix.multiplySparse (gloo for the gathers, so both ranks may share one GPU): A's and
B's rows are dealt to the ranks interleaved; B is gathered to every rank and each rank multiplies its own rows of A.
Each rank saves its COO entries for the caller to compare with the one-rank result bit for bit."""
import os
import sys
from pathlib import Path

import numpy as np
import torch.distributed as dist

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import marlin_b200 as mb
from marlin_b200.matrix.sparse_matrix import SparseVector


def data():
    rng = np.random.default_rng(21)
    K, n, m = 700, 5000, 300
    B = [(k, np.sort(rng.choice(n if k % 3 else 300, 1 + k % 97, replace=False)), None) for k in range(K) if k % 11]
    B = [(k, ix, rng.standard_normal(ix.size)) for k, ix, _ in B]
    A = []
    for i in range(m):
        cnt = int(rng.integers(0, 120 if i % 10 else 600))
        ix = np.sort(rng.choice(K, cnt, replace=False))
        A.append((i, ix, rng.standard_normal(cnt)))
    return A, B, m, K, n


def _mine(rows, rank, ws, n_rows, n_cols):
    return mb.SparseVecMatrix([(i, SparseVector(n_cols, ix, v)) for t, (i, ix, v) in enumerate(rows) if t % ws == rank],
                              n_rows, n_cols)


def main():
    dist.init_process_group("gloo")
    rank, ws = dist.get_rank(), dist.get_world_size()
    mb.Runtime.get()
    A, B, m, K, n = data()
    a, b = _mine(A, rank, ws, m, K), _mine(B, rank, ws, K, n)
    c = a.multiplySparse(b)
    dense = a.toDenseVecMatrix()
    assert a.elementsCount() == m and b.elementsCount() == len(B), (a.elementsCount(), b.elementsCount())
    np.savez(os.environ["SPVEC_WORKER_OUT"] + f".{rank}.npz", r=c.rows, c=c.cols, v=c.values, dense_rows=len(dense.ids))
    try:
        a.multiplySparse(_mine(B, rank, ws, K + 1, n))
        raise AssertionError("no error")
    except mb.MarlinArgumentError as e:
        assert "does not match" in str(e), str(e)
    print(f"rank {rank} mismatch raised")
    # a row id held by both ranks fails every rank before the exchange
    dup = mb.SparseVecMatrix([(5, SparseVector(K, [1], [1.0]))], m, K)
    try:
        dup.multiplySparse(b)
        raise AssertionError("no error")
    except mb.MarlinArgumentError as e:
        assert "repeated row id 5" in str(e), str(e)
    try:
        a.multiplySparse(mb.SparseVecMatrix([(3, SparseVector(n, [1], [1.0]))], K, n))
        raise AssertionError("no error")
    except mb.MarlinArgumentError as e:
        assert "repeated row id 3" in str(e), str(e)
    print(f"rank {rank} duplicate raised")
    dist.barrier()
    dist.destroy_process_group()
    print(f"rank {rank} spvec ok")


if __name__ == "__main__":
    main()

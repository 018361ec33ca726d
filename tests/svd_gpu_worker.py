"""Two-rank worker (NCCL, one process per GPU) for DenseVecMatrix.computeSVD: interleaved row ids, one rank without rows;
s and V must be bitwise equal across ranks and agree with the one-rank result."""
import os
import sys
from pathlib import Path

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import marlin_b200 as mb


def main():
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    rank, ws = dist.get_rank(), dist.get_world_size()
    mb.Runtime.get()
    rng = np.random.default_rng(11)
    A = rng.standard_normal((3000, 129))
    ref = mb.SubMatrix(A).gramian()                          # one-rank reference, computed on each rank
    w_ref, v_ref = ref.symmetricEigen()
    s_ref = np.sqrt(np.abs(w_ref))[:12]
    for layout in ("interleaved", "one-rank-empty"):
        if layout == "interleaved":
            rows = [(i, A[i]) for i in range(A.shape[0]) if i % ws == rank]
        else:
            rows = [(i, A[i]) for i in range(A.shape[0])] if rank == 1 else []
        mat = mb.DenseVecMatrix(rows, A.shape[0], A.shape[1])
        U, s, V = mat.computeSVD(12, computeU=True)
        got = [None] * ws
        dist.all_gather_object(got, (s, V))
        for s2, V2 in got:
            assert np.array_equal(s2, s) and np.array_equal(V2, V), layout
        assert np.abs(s - s_ref).max() <= 1e-10 * s_ref[0], layout
        assert np.abs(np.abs(V.T @ v_ref.toBreeze()[:, :12]) - np.eye(12)).max() <= 1e-8, layout
        full = U.toBreeze()
        assert full.shape == A.shape[:1] + (12,)
        assert np.abs(full - A @ V / s).max() <= 1e-10 * np.abs(A @ V / s).max(), layout
        mine = set(int(i) for i in U.ids)
        assert mine == set(i for i, _ in rows), layout
    dist.barrier()
    dist.destroy_process_group()
    print(f"rank {rank} svd ok")


if __name__ == "__main__":
    main()

"""Multi-GPU worker (NCCL, one process per GPU): the sharded multiply path end to end against the oracle."""
import os
import sys
from pathlib import Path

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import marlin_b200 as mb
from marlin_b200 import comm
from oracle import reference_model as rm


def main():
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    rank, ws = dist.get_rank(), dist.get_world_size()
    mb.Runtime.get()
    rng = np.random.default_rng(0)
    # ---- BlockMatrix x BlockMatrix for several grids (ragged blocks), incl. k-splits that force a cross-rank reduce
    for (M, K, N, m, k, n) in [(64, 64, 64, 2, 2, 2), (100, 90, 70, 2, 2, 2), (96, 200, 64, 1, 2, 1), (130, 120, 110, 3, 2, 2),
                               (256, 256, 256, 4, 4, 4), (64, 512, 64, 1, 8, 1)]:
        A, B = rng.random((M, K)) * 2 - 1, rng.random((K, N)) * 2 - 1
        oa = rm.DenseVecMatrix(list(enumerate(A))).to_block_matrix(m, k)
        ob = rm.DenseVecMatrix(list(enumerate(B))).to_block_matrix(k, n)
        mk = lambda obm: mb.BlockMatrix([(mb.BlockID(r, c), mb.SubMatrix(blk)) for (r, c), blk in obm.blocks
                                         if comm.elem_owner(r, c, obm.num_blks_by_col(), ws) == rank],
                                        obm.num_rows(), obm.num_cols(), obm.num_blks_by_row(), obm.num_blks_by_col())
        ga, gb = mk(oa), mk(ob)
        ref = oa.multiply(ob, gemm="f2j").to_breeze()
        for rep in range(3):            # repeated epochs reuse the staging slots / flags of the peer-memory transport
            got = ga.multiply(gb)
            full = got.toBreeze()
            err = (np.abs(full - ref) / (np.abs(A) @ np.abs(B))).max()
            assert err <= 1e-10, (M, K, N, m, k, n, rep, err)
        # every C tile lives on exactly one rank, and the owner map agrees
        mine = {(b.row, b.column) for b, _ in got.blocks}
        for (i, j) in mine:
            assert got.owner(i, j) == rank
        # transpose and add stay block-local; re-grid moves pieces between GPUs
        assert np.array_equal(ga.transpose().toBreeze(), A.T)
        assert np.array_equal(ga.add(ga).toBreeze(), A + A)
        assert np.array_equal(ga.toBlockMatrix(k, m).toBreeze(), A)
        assert np.array_equal(ga.toDenseVecMatrix().toBreeze(), A)
        assert abs(ga.sum() - A.sum()) <= 1e-9 * abs(A).sum()
    # ---- bf16 tiles (config-5 path): C-stationary (4,4,4) and a k-split that reduces fp32 partials across ranks
    from marlin_b200 import _native as nat
    # 1000 on a 3 x 3 grid: 334- and 332-row blocks packed with ld = rows, so their operands are staged before the TMA
    for (n_, g_, kgrid) in [(512, 4, None), (256, None, (1, 4, 1)), (1000, 3, None)]:
        if kgrid is None:
            Ab = mb.MTUtils.randomBlockMatrix(None, n_, n_, g_, g_, seed=21, dtype=nat.MB_BF16)
            Bb = mb.MTUtils.randomBlockMatrix(None, n_, n_, g_, g_, seed=22, dtype=nat.MB_BF16)
        else:
            Ab = mb.MTUtils.randomBlockMatrix(None, n_, 4 * n_, kgrid[0], kgrid[1], seed=23, dtype=nat.MB_BF16)
            Bb = mb.MTUtils.randomBlockMatrix(None, 4 * n_, n_, kgrid[1], kgrid[2], seed=24, dtype=nat.MB_BF16)
        Cb = Ab.multiply(Bb)
        ref = Ab.toBreeze() @ Bb.toBreeze()
        assert (np.abs(Cb.toBreeze() - ref) / ref).max() <= 1e-4
    # ---- DenseVecMatrix: row shards, broadcast multiply (tall-skinny path), rows -> blocks -> multiply
    M, K, N = 301, 64, 48
    A, B = rng.random((M, K)), rng.random((K, N))
    lo, hi = (rank * M) // ws, ((rank + 1) * M) // ws
    ga = mb.DenseVecMatrix([(i, A[i]) for i in range(lo, hi)])
    gb = mb.DenseVecMatrix([(i, B[i]) for i in range(K) if i % ws == rank])
    denom = np.abs(A) @ np.abs(B)
    assert (np.abs(ga.multiply(B).toBreeze() - A @ B) / denom).max() <= 1e-10
    assert (np.abs(ga.multiply(gb, 2 * ws).toBreeze() - A @ B) / denom).max() <= 1e-10       # chooser -> broadcast branch
    assert (np.abs(ga.multiply(gb, (2, 2, 2)).toBreeze() - A @ B) / denom).max() <= 1e-10    # rows -> blocks across GPUs
    assert np.array_equal(ga.transpose().toBreeze(), A.T)
    assert np.array_equal(ga.add(ga).toBreeze(), 2 * A)
    # ---- vector side: pieces on rank id mod G, block x piece on the block's GPU, row partials reduced across ranks
    S = 600
    Asq, xv = rng.random((S, S)), rng.random(S)
    gsq = mb.DenseVecMatrix([(i, Asq[i]) for i in range(S) if i % ws == rank]).toBlockMatrix(3, 2)
    dvec = mb.DistributedVector.fromVector(None, xv, 2)
    dsq = np.abs(Asq) @ np.abs(xv)
    assert (np.abs(gsq.multiply(dvec).toBreeze() - Asq @ xv) / dsq).max() <= 1e-10
    gcol = mb.DenseVecMatrix([(i, Asq[i]) for i in range(S) if i % ws == rank])
    assert (np.abs(gcol.multiply(xv, 3).toBreeze() - Asq @ xv) / dsq).max() <= 1e-10
    assert (np.abs(gcol.multiply(xv) - Asq @ xv) / dsq).max() <= 1e-10
    d1 = mb.DistributedVector.fromVector(None, xv, 4)
    assert abs(d1.transpose().multiply(d1) - xv @ xv) <= 1e-10 * (xv @ xv)
    assert np.array_equal(d1.multiply(d1.transpose()).toBreeze(), np.outer(xv, xv))
    # generators are partition-deterministic regardless of the number of GPUs
    g = mb.MTUtils.randomDenVecMatrix(None, 50, 7, numPartitions=4, seed=11)
    assert np.array_equal(g.toBreeze(), rm.random_den_vec_matrix(50, 7, 4, seed=11).to_breeze())
    gbm = mb.MTUtils.randomBlockMatrix(None, 33, 21, 3, 2, seed=12)
    assert np.array_equal(gbm.toBreeze(), rm.random_block_matrix(33, 21, 3, 2, seed=12).to_breeze())
    dist.barrier()
    torch.cuda.synchronize()
    dist.destroy_process_group()
    print(f"rank {rank} ok transport={os.environ.get('MARLIN_B200_TRANSPORT', 'p2p')} "
          f"mesh={'yes' if __import__('marlin_b200.peer', fromlist=['PeerMesh']).PeerMesh._instance is not None else 'no'}")


if __name__ == "__main__":
    main()

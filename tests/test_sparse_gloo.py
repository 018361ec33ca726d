"""world_size-2 gloo test (CPU) of the multi-rank host path of sparse tiles: packing, the nnz agreement, the exchange
and the global sparse flag (tests/sparse_dist_worker.py)."""
import os
import subprocess
import sys
from pathlib import Path

from tests.test_dist_gloo import _free_port

ROOT = Path(__file__).resolve().parents[1]


def test_sparse_tiles_over_gloo():
    port = _free_port()
    procs = []
    for rank in range(2):
        env = dict(os.environ, MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE="2",
                   LOCAL_RANK=str(rank), CUDA_VISIBLE_DEVICES="", OMP_NUM_THREADS="1")
        procs.append(subprocess.Popen([sys.executable, str(ROOT / "tests" / "sparse_dist_worker.py")], env=env,
                                      stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = []
    for p in procs:
        try:
            out, _ = p.communicate(timeout=240)
        except subprocess.TimeoutExpired:
            for q in procs:
                q.kill()
            raise
        outs.append(out)
    for rank, (p, out) in enumerate(zip(procs, outs)):
        assert p.returncode == 0, f"rank {rank} failed:\n{out}"
        assert f"rank {rank} ok" in out

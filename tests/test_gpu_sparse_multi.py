"""BlockMatrix.multiply with sparse blocks across two GPUs (tests/sparse_gpu_worker.py, one process per GPU over NCCL).
Skips on a machine with fewer than two GPUs."""
import os
import socket
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]


@pytest.mark.gpu
def test_two_rank_sparse_multiply():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), str(ROOT / "tests" / "sparse_gpu_worker.py")]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900, env=dict(os.environ))
    assert out.returncode == 0, out.stdout[-4000:]
    for r in range(2):
        assert f"rank {r} sparse ok" in out.stdout

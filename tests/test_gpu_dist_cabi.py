"""The multi-GPU multiply through the C ABI alone (mb_comm_init / mb_matmul_blocked_dist): N processes, ctypes + numpy,
no torch and no NCCL anywhere (tests/dist_cabi_worker.py).  With fewer GPUs than ranks the ranks share devices, so the
whole protocol also runs on a one-GPU box."""
import os
import subprocess
import sys
import uuid
from pathlib import Path

import pytest

from tests.harness import build_cpp

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]


def _run(world, ndev, slow, timeout=900, big=0, big_fused=0, extra_env=None):
    session = uuid.uuid4().hex[:16]
    env = dict(os.environ, MARLIN_B200_TIMEOUT_S="90", MARLIN_B200_DIST_SLOW="1" if slow else "0", MB_BIG=str(big),
               CUDA_DEVICE_MAX_CONNECTIONS="32", MB_BIG_FUSED=str(big_fused), **(extra_env or {}))
    procs = [subprocess.Popen([sys.executable, str(ROOT / "tests" / "dist_cabi_worker.py"), str(r), str(world), session, str(ndev)],
                              stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env) for r in range(world)]
    outs = []
    for p in procs:
        try:
            out, _ = p.communicate(timeout=timeout)
        except subprocess.TimeoutExpired:
            for q in procs:
                q.kill()
            raise
        outs.append((p.returncode, out))
    for r, (rc, out) in enumerate(outs):
        assert rc == 0 and f"cabi rank {r}/{world} ok" in out, f"rank {r}:\n{out[-3000:]}"
    return outs


@pytest.mark.parametrize("slow", [False, True])
def test_dist_multiply_cabi_two_ranks(slow):
    """fast = the grouped DMMA kernel with band flags, two launches per rank with the fused reduce-scatter's exchange flags
    between them; slow = staged partials and
    per-tile launches (the path bf16 / transposed tiles take), forced here for fp64 so both are checked bit-for-tolerance."""
    import torch
    ndev = torch.cuda.device_count()
    _run(2, min(2, ndev), slow)


def test_dist_multiply_cabi_all_gpus():
    import torch
    ndev = torch.cuda.device_count()
    if ndev < 3:
        pytest.skip("needs >= 3 GPUs (the 2-rank case runs everywhere)")
    _run(min(ndev, 8), min(ndev, 8), False)


def test_dist_host_path_bench_size_pinned():
    """The end-to-end entry at a bench-like size (8192^2, 2x2 grid: 4096^2 tiles, four bands each) with PINNED shared host
    tiles: all copies are asynchronous, so each rank's grouped GEMM is resident and spinning on band flags long before the
    first band lands — the situation in which a flag written by a kernel (instead of a stream memory operation) deadlocks."""
    import torch
    ndev = torch.cuda.device_count()
    if ndev < 2:
        # two processes time-slicing ONE GPU make no useful progress here: each context's resident GEMM spins through its
        # time slices while the other context's copies and memory operations wait for theirs
        pytest.skip("needs 2 GPUs (the small host-path cases of the two-rank test run on one)")
    outs = _run(2, 2, False, big=8192)
    assert "big e2e parity" in outs[0][1]


def test_fused_reduce_scatter_full_size_back_to_back():
    """8192^2 with the contraction split over two GPUs, six multiplies queued back to back: the first launch's epilogues
    store the peer's half over NVLink, and the flag that announces it, a stream memory operation after that launch, must
    not overtake those stores.  Freivalds on the first and the last result."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    outs = _run(2, 2, False, big_fused=8192)
    assert "big fused" in "".join(o for _, o in outs)


def build_cpp_rank_program() -> Path:
    return build_cpp("dist_multiply", opt="-O2", extra=("-Wextra",))


@pytest.mark.parametrize("dims", [(700, 528, 900, 2, 3, 2), (512, 1024, 512, 1, 2, 1), (701, 530, 899, 2, 3, 2)],
                         ids=["even-blocks-grouped-launch", "k-split-reduce-scatter", "ragged-odd-general-path"])
def test_compiled_host_mirror_multiplies_across_two_ranks(dims):
    """The C++ host mirror's BlockMatrix.multiply(other, comm) (include/marlin_b200.hpp -> mb_matmul_blocked_dist) from a
    compiled rank program, two processes (sharing the GPU on a one-GPU box): integer-valued inputs, so the C blocks are
    compared with the host product EXACTLY.  Runs last of all (tests/conftest.py)."""
    import torch
    exe = build_cpp_rank_program()
    ndev = min(2, torch.cuda.device_count())
    session = uuid.uuid4().hex[:16]
    env = dict(os.environ, MARLIN_B200_TIMEOUT_S="90", CUDA_DEVICE_MAX_CONNECTIONS="32")
    procs = [subprocess.Popen([str(exe), str(r), "2", session, str(ndev)] + [str(d) for d in dims], stdout=subprocess.PIPE,
                              stderr=subprocess.STDOUT, text=True, env=env) for r in range(2)]
    outs = []
    for p in procs:
        try:
            out, _ = p.communicate(timeout=600)
        except subprocess.TimeoutExpired:
            for q in procs:
                q.kill()
            raise
        outs.append((p.returncode, out))
    for r, (rc, out) in enumerate(outs):
        assert rc == 0 and f"cpp rank {r}/2 ok" in out, f"rank {r}:\n{out[-3000:]}"

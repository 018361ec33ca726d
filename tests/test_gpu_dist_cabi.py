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


def _run_exact(group, world=2, timeout=600):
    """The exact-integer rank program (tests/dist_exact_worker.py) on `world` ranks for one case group of
    tests/dist_exact_cases.py; every rank must report every case of the group and end with its "ok" line."""
    import torch
    from tests import dist_exact_cases as dc
    ndev = min(world, torch.cuda.device_count())
    session = uuid.uuid4().hex[:16]
    env = dict(os.environ, MARLIN_B200_TIMEOUT_S="90", MARLIN_B200_DIST_SLOW="0", CUDA_DEVICE_MAX_CONNECTIONS="32")
    procs = [subprocess.Popen([sys.executable, str(ROOT / "tests" / "dist_exact_worker.py"), group, str(r), str(world), session, str(ndev)],
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
    names = [c.name for c in dc.group(group)] + ([c.name for c in dc.group("queued")] if group == "fresh" else [])
    for r, (rc, out) in enumerate(outs):
        assert rc == 0 and f"exact rank {r}/{world} ok group={group}" in out, f"rank {r}:\n{out[-3000:]}"
        for name in names:
            assert f"case {name}: rank {r} " in out or f"host error {name}: " in out, f"rank {r} did not report {name}:\n{out[-3000:]}"
    return [out for _, out in outs]


def test_dist_exact_path_limits():
    """Every limit of the fast path (k segments, distinct A and B operand tiles, entries per rank, plain tiles) exactly
    at and one past it, each result compared with == and each call's path named by its launch count."""
    _run_exact("limits")


def test_dist_exact_column_split_and_bands():
    """Fused C tiles N in {1, 100, 128, 129, 255, 256, 257, 385} wide (the owner reduces [0, half_cols(N)), the partner
    the rest), and operand extents 1023 / 1024 / 1025 / 1537 (1, 4, 3 and 4 readiness bands)."""
    _run_exact("split")


def test_dist_exact_fresh_operands_every_call():
    """One communicator, new operands and NaN-refilled C tiles every call, plans alternating (fused, (2,2,2), a larger
    tile that grows the staging buffer and smaller ones that reuse it, one staged-path call), more calls than the
    mailbox ring has slots; then six calls queued without a host synchronisation, checked after the last."""
    _run_exact("fresh")


def test_dist_exact_c_views():
    """The owner's C tile as a slice of a sentinel-filled parent: even ld and a 16-byte aligned offset (fast path: the
    partner's epilogue writes its reduced half into the view remotely) and odd ld (general path).  Exact results, and
    every parent element outside the view keeps its bits."""
    _run_exact("views")


def test_dist_exact_bf16():
    """bf16 tiles (general path, fp32 C) with integer operands |x| <= 256 whose sums stay below 2^24: exact."""
    _run_exact("bf16")


def test_dist_exact_special_values():
    """A NaN and a -Inf in A rows and a +Inf in a B column, all computed by the rank that does not own the fused C tile:
    each affected entry's class (NaN, +Inf, -Inf) follows IEEE arithmetic and every other entry is exact."""
    _run_exact("special")


def test_dist_exact_host_entry():
    """mb_matmul_blocked_dist_host at the band edges: 1 x 1, 3 x 3 and 4 x 4 checkerboards of sub-blocks, a one-wide
    last band; fresh data each rep and host C refilled with 0xFF each time."""
    _run_exact("host")


def test_dist_exact_host_limits():
    """The host entry's feasibility limits at and one past (uploads per rank, k, sub-blocks per rank): one past returns
    MB_ERR_UNSUPPORTED on every rank with the same message, and the next call on the same communicator is exact."""
    outs = _run_exact("host_limits")
    errors = [sorted(line for line in out.splitlines() if line.startswith("host error ")) for out in outs]
    assert errors[0] and all(e == errors[0] for e in errors), errors


def test_dist_exact_three_holders():
    """A C tile with three holders: staged partials added by the owner in holder order, on the fast and the general
    path, exact."""
    import torch
    if torch.cuda.device_count() < 3:
        pytest.skip("needs >= 3 GPUs (the 2-rank cases run everywhere)")
    _run_exact("holders3", world=3)


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

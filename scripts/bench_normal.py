"""Time the StandardNormalGenerator fill (mb_fill_normal) on the two shapes of the dense generators, against
mb_fill_uniform on the same blocks and torch.randn(float64) as a speed yardstick (torch uses its own stream and a
different generator, so it only says how fast a Gaussian fill can be).

Per shape: a 1048576 x 1024 row shard (rows one after another) and a 16384 x 16384 column-major block.
  * mb_fill_normal end to end: host clock around the blocking call (its stream synchronisations included), best of
    --repeats after --warmup calls;
  * each pass on its own (count, scan, write) and the uniform kernels: kernel durations from a torch.profiler run of
    one more call each, after the timed runs;
  * mb_fill_uniform: host clock around the call and a synchronisation; torch.randn: CUDA events.
Values/s and the write bandwidth 8n/t are reported, the latter against the H100 SXM's 3.35 TB/s.  A seeded prefix and a
far slice of the timed output are checked bit for bit against tests/normal_oracle.py.  The card's name, power limit and
clocks are read in the same run.  Prints one JSON line per shape.

    python scripts/bench_normal.py [--shapes 1048576x1024:rows,16384x16384:cols] [--repeats 5] [--warmup 2]
"""
import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import marlin_b200 as mb
from marlin_b200 import _native as nat
from tests import normal_oracle as no

HBM = 3.35e12
SEED = 20261017


def host_best(fn, repeats, warmup):
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        times.append(time.perf_counter() - t0)
    return min(times)


def event_best(fn, repeats, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(repeats):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        fn()
        t1.record()
        torch.cuda.synchronize()
        times.append(t0.elapsed_time(t1) / 1e3)
    return min(times)


def kernel_times(fn, names):
    """Total device seconds per kernel whose name contains one of `names`, for one call of fn."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {n: 0.0 for n in names}
    for ev in prof.events():
        for n in names:
            if n in ev.name and ev.device_type == torch.autograd.DeviceType.CUDA:
                out[n] += ev.device_time_total / 1e6 if hasattr(ev, "device_time_total") else ev.cuda_time_total / 1e6
    return out


def check_oracle(got_flat, n, chunk=1 << 24):
    """A seeded prefix and a far slice of fill order against the oracle."""
    k = 1 << 16
    ok = np.array_equal(got_flat(0, k).view(np.uint64), no.normal_stream(SEED, k)[0].view(np.uint64))
    # the far slice starts at the first value of attempt a_far, about 90 % into the fill: 2 * (accepted attempts before it)
    a_far, before = int(0.9 * n / 2 * 4 / np.pi) // chunk * chunk, 0
    for a in range(0, a_far, chunk):
        before += int(no.accepted_attempts(SEED, chunk, a).sum())
    m = min(k, n - 2 * before)
    want = no.normal_stream(SEED, m, first_attempt=a_far)[0]
    return ok and np.array_equal(got_flat(2 * before, m).view(np.uint64), want.view(np.uint64)), 2 * before


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="1048576x1024:rows,16384x16384:cols")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    rt = mb.Runtime.get()
    lib, ctx = rt.lib, rt.ctx
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm,clocks.mem", "--format=csv,noheader",
                           "-i", str(rt.device_index)], stdout=subprocess.PIPE, text=True).stdout.strip()
    for spec in a.shapes.split(","):
        shape, order = spec.split(":")
        m, n = (int(v) for v in shape.split("x"))
        total = m * n
        row_major = 1 if order == "rows" else 0
        buf = torch.empty(total, dtype=torch.float64, device=rt.device)
        blk = nat.c_blk()
        # rows: element (r, c) at r * n + c (a row shard); cols: at r + c * m (a column-major block); fill order = storage
        nat.check(lib.mb_block_wrap(ctx, C.c_void_p(buf.data_ptr()), 0, m, n, n if row_major else m, row_major, nat.MB_F64,
                                    C.byref(blk)))
        rt.sync_stream()
        normal = lambda: nat.check(lib.mb_fill_normal(ctx, blk, SEED, 0.0, 1.0, row_major, None))

        def uniform():
            nat.check(lib.mb_fill_uniform(ctx, blk, SEED, 0, 0.0, 1.0, row_major))
            nat.check(lib.mb_synchronize(ctx))

        t_normal = host_best(normal, a.repeats, a.warmup)
        normal()
        nat.check(lib.mb_synchronize(ctx))
        host = lambda start, cnt: buf[start:start + cnt].cpu().numpy()
        ok, far = check_oracle(host, total)
        t_uniform = host_best(uniform, a.repeats, a.warmup)
        t_randn = event_best(lambda: torch.randn(total, dtype=torch.float64, device=rt.device, out=buf), a.repeats, a.warmup)
        passes = kernel_times(normal, ["normal_count_kernel", "normal_scan_kernel", "normal_write_kernel"])
        upasses = kernel_times(uniform, ["fill_uniform"])
        nat.check(lib.mb_block_free(ctx, blk))
        del buf
        torch.cuda.empty_cache()
        rec = {
            "shape": spec, "values": total, "card": card,
            "normal_ms": t_normal * 1e3, "normal_values_per_s": total / t_normal, "normal_write_TBps": 8 * total / t_normal / 1e12,
            "count_ms": passes["normal_count_kernel"] * 1e3, "scan_ms": passes["normal_scan_kernel"] * 1e3,
            "write_ms": passes["normal_write_kernel"] * 1e3,
            "write_pass_TBps": 8 * total / max(passes["normal_write_kernel"], 1e-12) / 1e12,
            "uniform_ms": t_uniform * 1e3, "uniform_kernel_ms": upasses["fill_uniform"] * 1e3,
            "uniform_TBps": 8 * total / t_uniform / 1e12,
            "torch_randn_ms": t_randn * 1e3, "torch_randn_TBps": 8 * total / t_randn / 1e12,
            "hbm_share_normal": 8 * total / t_normal / HBM,
            "oracle_prefix_and_far_slice_match": bool(ok), "far_slice_first_value": far,
        }
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()

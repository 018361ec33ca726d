"""Time DenseVecMatrix.norm's kernel (mb_block_norm) on one fp64 row shard, with device events, against
torch.linalg.matrix_norm on the same tensor.

For each shape and mode: warm-up calls, then the best of --repeats timed calls.  GB/s counts one read of the shard.
The card's name and power limit are read in the same run.  Prints one JSON line per shape and mode.

    python scripts/bench_norm.py [--shapes 1048576x1024,4194304x256] [--repeats 7] [--warmup 3]
"""
import argparse
import ctypes as C
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import marlin_b200 as mb
from marlin_b200 import _native as nat

MODES = {"1": (nat.MB_NORM_ONE, 1), "inf": (nat.MB_NORM_INF, float("inf")), "fro": (nat.MB_NORM_FRO, "fro")}


def best_ms(fn, repeats, warmup):
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
        times.append(t0.elapsed_time(t1))
    return min(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="1048576x1024,4194304x256")
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    rt = mb.Runtime.get()
    lib, ctx = rt.lib, rt.ctx
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(rt.device_index)],
                          stdout=subprocess.PIPE, text=True).stdout.strip()
    for shape in a.shapes.split(","):
        m, n = (int(v) for v in shape.split("x"))
        x = torch.rand(m, n, dtype=torch.float64, device=rt.device)
        blk = mb.SubMatrix(buf=x.view(-1), rows=m, cols=n, ld=n, is_transpose=True)
        col = mb.SubMatrix.empty(n, 1, nat.MB_F64)
        out = np.zeros(3)
        gb = m * n * 8 / 1e9
        for mode, (kind, ord_) in MODES.items():
            rt.sync_stream()
            call = lambda: nat.check(lib.mb_block_norm(ctx, blk.handle(), kind, col.handle(), out.ctypes.data_as(nat.c_dp)))
            ours = best_ms(call, a.repeats, a.warmup)
            theirs = best_ms(lambda: torch.linalg.matrix_norm(x, ord=ord_), a.repeats, a.warmup)
            print(json.dumps({"shape": [m, n], "mode": mode, "ms": round(ours, 4), "GBps": round(gb / ours * 1e3, 1),
                              "torch_ms": round(theirs, 4), "torch_GBps": round(gb / theirs * 1e3, 1), "card": card}),
                  flush=True)
        del x, blk


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Time per iteration of DenseVecMatrix.lr on one GPU: the fused gradient kernel looped on the device (mb_lr_train)
against the two-pass composition a user could build from the existing ops (margins by gemv N over the row shard, the
sigmoid on the host, the gradient by gemv T), at 1048576 x 1024 and 4194304 x 256 fp64 (8 GiB each).

Effective GB/s counts one read of the shard per iteration (8 m n bytes), the least any gradient step must move, for both
paths.  DRAM bytes are not measured here (Nsight Compute is not used).  Each window is timed with a host clock around work
that ends in a device synchronise, after a warm-up of the same shape; the card's name, power limit and SM clock are read
with nvidia-smi in the same run and printed beside the numbers.  Prints one JSON document (also written to --out).

  python scripts/bench_lr.py [--iters 20] [--rounds 3] [--only 1048576x1024] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

SHAPES = {"1048576x1024": (1048576, 1024), "4194304x256": (4194304, 256)}


def smi(query: str) -> str:
    out = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader", "-i", "0"], stdout=subprocess.PIPE,
                         stderr=subprocess.DEVNULL, text=True)
    return out.stdout.strip()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--only", default="")
    ap.add_argument("--out", default="")
    args = ap.parse_args()

    import numpy as np
    import torch
    import marlin_b200 as mb
    from marlin_b200 import _native as nat

    if not torch.cuda.is_available():
        raise SystemExit("bench_lr needs a CUDA device: there is nothing to measure without one")
    rt = mb.Runtime.get()
    card = {"gpu": smi("name"), "power_limit": smi("power.limit"), "clocks_max_sm": smi("clocks.max.sm")}
    results = []
    for name, (m, n) in SHAPES.items():
        if args.only and name not in args.only.split(","):
            continue
        gen = torch.Generator(device="cuda").manual_seed(1)
        X = torch.randn(m * n, dtype=torch.float64, device="cuda", generator=gen) / 8
        X.view(m, n)[:, 0] = (torch.rand(m, device="cuda", generator=gen) < 0.5).double()
        shard = mb.SubMatrix(buf=X, rows=m, cols=n, ld=n, is_transpose=True)
        w_out = np.zeros(n)

        def fused(iters: int) -> None:
            rt.sync_stream()
            nat.check(rt.lib.mb_lr_train(rt.ctx, shard.handle(), m, 1.0, iters, w_out.ctypes.data_as(nat.c_dp)))

        wv = mb.SubMatrix.zeros(n, 1, nat.MB_F64)
        margins = mb.SubMatrix.empty(m, 1, nat.MB_F64)
        grad = mb.SubMatrix.empty(n, 1, nat.MB_F64)
        label = X.view(m, n)[:, 0].cpu().numpy()

        def composed(iters: int) -> None:
            w = np.zeros(n)
            for i in range(1, iters + 1):
                wv.buf[:n].copy_(torch.from_numpy(w))
                shard.multiply(wv, out=margins)                                     # gemv N: one read of the shard
                dot = margins.buf[:m].cpu().numpy()
                g = 1.0 / (1.0 + np.exp(-dot)) - label                              # host sigmoid
                gd = mb.SubMatrix(g.reshape(-1, 1), device=X.device)
                shard.t.multiply(gd, out=grad)                                      # gemv T: a second read
                w = w - grad.buf[:n].cpu().numpy() * (1.0 / m / np.sqrt(i))
            torch.cuda.synchronize()

        row = {"shape": name, "bytes_per_iteration": 8 * m * n, "fused_ms": [], "composed_ms": [], "sm_clock": []}
        fused(2)
        composed(2)
        for _ in range(args.rounds):
            for label_, fn in (("fused_ms", fused), ("composed_ms", composed)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn(args.iters)
                t1 = time.perf_counter()
                row[label_].append(1e3 * (t1 - t0) / args.iters)
            row["sm_clock"].append(smi("clocks.sm"))
        for k in ("fused", "composed"):
            best = min(row[f"{k}_ms"])
            row[f"{k}_GBps_best"] = round(row["bytes_per_iteration"] / (best * 1e-3) / 1e9, 1)
            row[f"{k}_ms"] = [round(v, 3) for v in row[f"{k}_ms"]]
        results.append(row)
        print(json.dumps(row), flush=True)
        del X, shard, margins, grad, wv
        torch.cuda.empty_cache()
    doc = {"card": card, "iters": args.iters, "results": results}
    print(json.dumps(doc))
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(doc, indent=1))


if __name__ == "__main__":
    main()

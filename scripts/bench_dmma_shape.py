#!/usr/bin/env python
"""A/B of the fp64 DMMA instruction shape in one process: the m16n8k4 kernels (default) against their m8n8k4 reference
instances (mb_set_dmma_reference), alternated --rounds times on each workload:

  headline   16384 x 16384 BlockMatrix multiply, 2 x 2 grid (bench.py's workload; grouped kernel)
  cfg1       4096 x 4096 multiply, one block (grouped kernel)
  cfg3       1048576 x 1024 row shard times 1024 x 1024 (gemm kernel <T,N>)
  gram1024   Gramian of a 1048576 x 1024 row shard (syrk kernel <N,T>, K split over partials)
  gram4096   Gramian of a 131072 x 4096 row shard (syrk kernel <N,T>)

Every window is timed with CUDA events after a warm-up of the same shape and lasts about --seconds; the SM clock, power
draw and active clock-event reasons are sampled with nvidia-smi during it and printed beside the rate, with the card's
name and power limit.  Prints one JSON document (also written to --out if given).

  python scripts/bench_dmma_shape.py [--rounds 3] [--seconds 1.0] [--only headline,cfg1] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import math
import statistics
import subprocess
import sys
import threading
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

Q = "clocks.sm,power.draw,clocks_event_reasons.sw_power_cap,clocks_event_reasons.hw_slowdown,clocks_event_reasons.sw_thermal_slowdown"


class Sampler:
    """nvidia-smi every 100 ms in the background; window(t0, t1) summarises the samples taken between two host times."""

    def __init__(self):
        self.samples = []
        self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={Q}", "--format=csv,noheader,nounits", "-lms", "100", "-i", "0"],
                                     stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        self.thread = threading.Thread(target=self._read, daemon=True)
        self.thread.start()

    def _read(self):
        for line in self.proc.stdout:
            f = [x.strip() for x in line.split(",")]
            try:
                self.samples.append((time.time(), float(f[0]), float(f[1]), [n for n, v in zip(("sw_power_cap", "hw_slowdown", "sw_thermal"), f[2:5])
                                                                             if v.lower().startswith("active")]))
            except (ValueError, IndexError):
                pass

    def window(self, t0, t1):
        s = [x for x in self.samples if t0 <= x[0] <= t1]
        if not s:
            return {"sm_mhz": None, "power_w": None, "reasons": [], "samples": 0}
        return {"sm_mhz": statistics.median(x[1] for x in s), "power_w": statistics.median(x[2] for x in s),
                "power_w_max": max(x[2] for x in s), "reasons": sorted({r for x in s for r in x[3]}), "samples": len(s)}

    def close(self):
        self.proc.terminate()
        try:
            self.proc.wait(timeout=3)
        except subprocess.TimeoutExpired:
            self.proc.kill()
            self.proc.wait()


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm,power.draw", "--format=csv,noheader",
                          "-i", "0"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True).stdout.strip()
    f = [x.strip() for x in out.split(",")]
    keys = ("name", "power_limit", "sm_max_clock", "sm_clock_idle", "power_draw_idle")
    return dict(zip(keys, f)) if len(f) == len(keys) else {"nvidia-smi": out}


def workloads(mb):
    """name -> (flop per call, make() returning the call's closure; the operands stay alive in the closure)."""
    from marlin_b200.matrix.sub_matrix import SubMatrix

    def blocked(n, g):
        A = mb.MTUtils.randomBlockMatrix(None, n, n, g, g, seed=42)
        B = mb.MTUtils.randomBlockMatrix(None, n, n, g, g, seed=43)
        return lambda: A.multiply(B)

    def rowsharded():
        A = mb.MTUtils.randomDenVecMatrix(None, 1048576, 1024, numPartitions=1, seed=42)
        B = SubMatrix(mb.MTUtils.randomBlockMatrix(None, 1024, 1024, 1, 1, seed=43).toBreeze())
        return lambda: A.multiply(B)

    def gram(m, n):
        A = mb.MTUtils.randomDenVecMatrix(None, m, n, numPartitions=1, seed=42)
        return lambda: A.data.gramian()

    return {
        "headline": (2.0 * 16384 ** 3, lambda: blocked(16384, 2)),
        "cfg1": (2.0 * 4096 ** 3, lambda: blocked(4096, 1)),
        "cfg3": (2.0 * 1048576 * 1024 * 1024, rowsharded),
        # the Gramian's useful work: the lower triangle and diagonal of G, n(n+1)/2 dot products of length m
        "gram1024": (1048576 * 1024.0 * 1025, lambda: gram(1048576, 1024)),
        "gram4096": (131072 * 4096.0 * 4097, lambda: gram(131072, 4096)),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--only", default=None)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    import marlin_b200 as mb
    rt = mb.Runtime.get()
    result = {"card": card(), "rounds": args.rounds, "workloads": {}}
    sampler = Sampler()
    try:
        for name, (flop, make) in workloads(mb).items():
            if args.only and name not in args.only.split(","):
                continue
            call = make()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            steps = {}
            for ref in (False, True):                      # warm up both kernels and size the windows
                rt.set_dmma_reference(ref)
                for _ in range(2):
                    out = call()
                    del out
                torch.cuda.synchronize()
                e0.record()
                out = call()
                e1.record()
                torch.cuda.synchronize()
                del out
                steps[ref] = max(3, math.ceil(args.seconds * 1e3 / max(e0.elapsed_time(e1), 1e-3)))
            runs = {"m16n8k4": [], "m8n8k4_reference": []}
            for _ in range(args.rounds):
                for ref in (True, False):
                    rt.set_dmma_reference(ref)
                    n = max(steps.values())
                    out = call()
                    torch.cuda.synchronize()
                    t0 = time.time()
                    e0.record()
                    for _ in range(n):
                        del out
                        out = call()
                    e1.record()
                    torch.cuda.synchronize()
                    t1 = time.time()
                    del out
                    ms = e0.elapsed_time(e1) / n
                    runs["m8n8k4_reference" if ref else "m16n8k4"].append(
                        {"ms": ms, "tflops": flop / (ms * 1e-3) / 1e12, "steps": n, **sampler.window(t0, t1)})
            rt.set_dmma_reference(False)
            best = {k: max(r["tflops"] for r in v) for k, v in runs.items()}
            worst = {k: min(r["tflops"] for r in v) for k, v in runs.items()}
            result["workloads"][name] = {"runs": runs, "best_tflops": best, "worst_tflops": worst,
                                         "speedup_worst_new_over_best_ref": worst["m16n8k4"] / best["m8n8k4_reference"]}
            print(name, json.dumps({k: [round(r["tflops"], 2) for r in v] for k, v in runs.items()}), flush=True)
            del call
            torch.cuda.empty_cache()
    finally:
        rt.set_dmma_reference(False)
        sampler.close()
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(text)


if __name__ == "__main__":
    main()

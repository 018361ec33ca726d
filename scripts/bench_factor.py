"""Dist-mode block LU / Cholesky / inverse on one GPU, and one step's trailing update as grouped launches vs per-block
`multiply` + `subtract`.  Prints one JSON document with the card's name and power limit.

    python scripts/bench_factor.py [--n 16384] [--bases 1000,2048] [--reps 3]

Rates count 2/3 n^3 (LU), 1/3 n^3 (Cholesky) and 2 n^3 (inverse) flops.  The update comparison alternates the two forms
on the same blocks (step 0 of an LU: every trailing block of an nb x nb grid) and checks that their outputs agree bit
for bit."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import marlin_b200 as mb
from marlin_b200.matrix import factorizations as fz


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip()
    return q or torch.cuda.get_device_name()


def timed(f):
    torch.cuda.synchronize()
    t = time.perf_counter()
    r = f()
    torch.cuda.synchronize()
    return time.perf_counter() - t, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=16384)
    ap.add_argument("--bases", default="1000,2048")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    mb.Runtime.get()
    n = a.n
    rng = np.random.default_rng(0)
    A = rng.standard_normal((n, n)) + n ** 0.5 * np.eye(n)
    M = mb.DenseVecMatrix(ids=np.arange(n), data=mb.SubMatrix(buf=torch.from_numpy(A.reshape(-1)).cuda(), rows=n, cols=n,
                                                               ld=n, is_transpose=True), nRows=n, nCols=n)
    S = mb.DenseVecMatrix(ids=np.arange(n), data=mb.SubMatrix(buf=torch.from_numpy((A @ A.T).reshape(-1)).cuda(), rows=n,
                                                              cols=n, ld=n, is_transpose=True), nRows=n, nCols=n)
    out = {"card": card(), "n": n, "factor": [], "update": []}
    flops = {"lu": 2 / 3 * n ** 3, "cholesky": 1 / 3 * n ** 3, "inverse": 2 * n ** 3}
    calls = {"lu": lambda b: M.luDecompose("dist", b), "cholesky": lambda b: S.choleskyDecompose("dist", b),
             "inverse": lambda b: M.inverse("dist", b)}
    for base in [int(x) for x in a.bases.split(",")]:
        for kind, f in calls.items():
            times = []
            for _ in range(a.reps):
                t, r = timed(lambda: f(base))
                del r
                times.append(t)
            best = min(times)
            out["factor"].append({"kind": kind, "base": base, "seconds": times, "tflops_best": flops[kind] / best / 1e12})
        # one step's trailing update on the grid of this base size
        nb, sub = fz.grid(n, base)
        blocks = {(r, c): mb.SubMatrix(A[r * sub:min(n, (r + 1) * sub), c * sub:min(n, (c + 1) * sub)], device="cuda")
                  for r in range(nb) for c in range(nb)}
        X = {r: blocks[(r, 0)] for r in range(1, nb)}
        Y = {c: blocks[(0, c)] for c in range(1, nb)}
        keys = [(r, c) for r in range(1, nb) for c in range(1, nb)]
        per_block, grouped = [], []
        for _ in range(a.reps):
            t, ref = timed(lambda: {k: blocks[k].subtract(X[k[0]].multiply(Y[k[1]])) for k in keys})
            per_block.append(t)
            cs = {k: blocks[k].copy() for k in keys}
            t, _ = timed(lambda: fz.schur_update([(cs[k], X[k[0]], Y[k[1]]) for k in keys]))
            grouped.append(t)
            same = all(torch.equal(cs[k].buf.view(torch.int64), ref[k].buf.view(torch.int64)) for k in keys)
            del ref, cs
        fl = 2.0 * sum(blocks[k].rows * blocks[k].cols * sub for k in keys)
        out["update"].append({"base": base, "blocks": len(keys), "per_block_s": per_block, "grouped_s": grouped,
                              "per_block_tflops_best": fl / min(per_block) / 1e12, "grouped_tflops_best": fl / min(grouped) / 1e12,
                              "bitwise_equal": bool(same)})
        del blocks, X, Y
    print(json.dumps(out))


if __name__ == "__main__":
    main()

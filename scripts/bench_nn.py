"""Time one NeuralNetwork iteration (mb_nn_step) on the GPU at MNIST's shape, with device events.

For each hidden width it alternates, in one process, the step with the hidden-weight gradient as K chunks of a grouped launch
(XT given) and the step with one transposed-A GEMM per block (no XT), and times the two large products on their own through
mb_dgemm_device: Z1 = X W1 per block, and X^T D1 per block as a transposed-A GEMM.  What is left of the chunked step after
Z1 is the fused backprop kernel (which reads Z1 once and writes D1 once: hidden_layer_bytes), the chunked hidden-weight
gradient and the two update kernels; they are not timed apart.
The card's name and power limit are read in the same run.  Prints one JSON line per width.

    python scripts/bench_nn.py [--rows 60000] [--blocks 8] [--widths 128,512] [--steps 20] [--warmup 3]
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

V = 784


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(steps):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=60000)
    ap.add_argument("--blocks", type=int, default=8)
    ap.add_argument("--widths", default="128,512")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    rt = mb.Runtime.get()
    lib, ctx = rt.lib, rt.ctx
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(rt.device_index)],
                          stdout=subprocess.PIPE, text=True).stdout.strip()
    rng = np.random.default_rng(0)
    sub = -(-a.rows // a.blocks)
    bounds = [(lo, min(a.rows, lo + sub)) for lo in range(0, a.rows, sub)]
    X = [mb.SubMatrix(rng.random((hi - lo, V)) * (rng.random((hi - lo, V)) < 0.2)) for lo, hi in bounds]
    XT = [x.transpose() for x in X]
    labels = []
    for lo, hi in bounds:
        y = rng.integers(0, 10, hi - lo).astype(np.int32)
        p = C.c_void_p()
        nat.check(lib.mb_nn_labels_upload(ctx, y.ctypes.data, len(y), C.byref(p)))
        labels.append(p)
    arr = lambda bl: (nat.c_blk * len(bl))(*[b.handle().value for b in bl])      # noqa: E731
    xs, xts = arr(X), arr(XT)
    ls = (C.c_void_p * len(labels))(*[p.value for p in labels])
    rt.sync_stream()
    for H in [int(w) for w in a.widths.split(",")]:
        W1, W2 = mb.SubMatrix(rng.normal(0, 0.2, (V, H))), mb.SubMatrix(rng.normal(0, 0.2, (H, 10)))
        Z = [mb.SubMatrix.zeros(x.rows + (x.rows & 1), H) for x in X]
        P = mb.SubMatrix.zeros(V, H)
        ptr = lambda s: C.c_void_p(s.buf.data_ptr())                             # noqa: E731

        def step(xt):
            nat.check(lib.mb_nn_step(ctx, xs, xt, ls, len(X), W1.handle(), W2.handle(), 1e-9))

        def gemm1():
            for x, z in zip(X, Z):
                nat.check(lib.mb_dgemm_device(ctx, b"N", b"N", x.rows, H, V, 1.0, ptr(x), x.ld, ptr(W1), V, 0.0, ptr(z), z.ld))

        def grad_transa():
            for x, z in zip(X, Z):
                nat.check(lib.mb_dgemm_device(ctx, b"T", b"N", V, H, x.rows, 1.0, ptr(x), x.ld, ptr(z), z.ld, 0.0, ptr(P), V))

        res = {"chunked_ms": [], "transa_ms": []}
        for _ in range(3):                                                       # alternate the two versions of the step
            res["chunked_ms"].append(timed(lambda: step(xts), a.steps, a.warmup))
            res["transa_ms"].append(timed(lambda: step(None), a.steps, a.warmup))
        t_chunk = min(res["chunked_ms"])
        t_g1, t_g2 = timed(gemm1, a.steps, a.warmup), timed(grad_transa, a.steps, a.warmup)
        flop = 2.0 * a.rows * V * H
        print(json.dumps({
            "card": card, "rows": a.rows, "blocks": len(X), "H": H, "step_chunked_ms": res["chunked_ms"],
            "step_transa_ms": res["transa_ms"], "gemm1_ms": t_g1, "gemm1_tflops": flop / t_g1 / 1e9,
            "w1_gradient_transa_ms": t_g2, "w1_gradient_transa_tflops": flop / t_g2 / 1e9,
            "chunked_step_after_gemm1_ms": t_chunk - t_g1, "hidden_layer_bytes": 2.0 * a.rows * H * 8}))
    for p in labels:
        lib.mb_nn_labels_free(ctx, p)


if __name__ == "__main__":
    main()

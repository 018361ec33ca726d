"""Time computeSVD's Lanczos path on the GPU: the one-pass A^T (A x) kernel (mb_block_gram_matvec) on fp64 row shards
against torch's `A.T @ (A @ x)` and the logistic-regression gradient kernel on the same shard, then
computeSVD(10, computeU=True, tol=1e-10, mode="dist-eigs") against the Gramian and Jacobi path, and on a matrix wider
than that path's 65535-column cap.

GB/s divides by the bytes the kernel's design needs (include/marlin_b200.h, csrc/eigs.cu): 8 m n for rows of at most 5118
columns, 16 m n + 16 n ceil(m / 8) for wider rows, plus 16 n per CTA partial and 16 n for x and y.  Kernel times are the
best of --repeats device-event windows after --warmup calls.  The card's name and power limit are read in the same run.
Prints one JSON line per measurement.

    python scripts/bench_eigs.py [--repeats 5] [--warmup 2] [--skip-svd]
"""
import argparse
import ctypes as C
import json
import math
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import marlin_b200 as mb
from marlin_b200 import _native as nat

RESIDENT_N = 5118


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


def design_bytes(m, n, sms):
    parts = min(sms, math.ceil(m / (min(32, 5120 // ((n + 2) & ~1)) if n <= RESIDENT_N else 8)))
    a = 8 * m * n if n <= RESIDENT_N else 16 * m * n + 16 * n * math.ceil(m / 8)
    return a + 16 * n * parts + 16 * n


def shard(m, n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    buf = torch.randn(m * n, dtype=torch.float64, device="cuda", generator=g)
    return buf, mb.SubMatrix(buf=buf, rows=m, cols=n, ld=n, is_transpose=True)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def bench_kernel(m, n, args, gpu, sms):
    rt = mb.Runtime.get()
    buf, blk = shard(m, n, m + n)
    x = mb.SubMatrix.empty(n, 1)
    x.buf.copy_(torch.randn(n, dtype=torch.float64, device="cuda"))
    y = mb.SubMatrix.empty(n, 1)
    rt.sync_stream()
    ms = best_ms(lambda: nat.check(rt.lib.mb_block_gram_matvec(rt.ctx, blk.handle(), x.handle(), y.handle(), 0)),
                 args.repeats, args.warmup)
    A = buf.view(m, n)
    xt = x.buf.view(n)
    torch_ms = best_ms(lambda: A.T @ (A @ xt), args.repeats, args.warmup)
    w = np.zeros(n)
    g = np.zeros(n)
    lr_ms = best_ms(lambda: nat.check(rt.lib.mb_lr_gradient(rt.ctx, blk.handle(), w.ctypes.data_as(nat.c_dp),
                                                            g.ctypes.data_as(nat.c_dp))), args.repeats, args.warmup)
    nbytes = design_bytes(m, n, sms)
    print(json.dumps({"kernel": "mb_block_gram_matvec", "m": m, "n": n, "ms": round(ms, 3), "design_bytes": nbytes,
                      "GB_per_s": round(nbytes / ms / 1e6, 1), "torch_AT_Ax_ms": round(torch_ms, 3),
                      "lr_gradient_ms": round(lr_ms, 3), "gpu": gpu}), flush=True)
    del A, buf, blk
    torch.cuda.empty_cache()


def bench_svd(m, n, k, args, gpu, old=True):
    buf, blk = shard(m, n, 7 * m + n)
    mat = mb.DenseVecMatrix(ids=np.arange(m), data=blk, nRows=m, nCols=n)
    out = {"call": f"computeSVD({k}, computeU=True, tol=1e-10, mode='dist-eigs')", "m": m, "n": n, "gpu": gpu}
    mat.computeSVD(k, computeU=True, mode="dist-eigs", tol=1e-10)          # warm-up: modules, pools
    torch.cuda.synchronize()
    t = time.perf_counter()
    U, s, V = mat.computeSVD(k, computeU=True, mode="dist-eigs", tol=1e-10)
    torch.cuda.synchronize()
    out["ms"] = round((time.perf_counter() - t) * 1e3, 1)
    out.update(mat.last_eigs_stats)
    out["s0"] = float(s[0])
    if old:
        torch.cuda.synchronize()
        t = time.perf_counter()
        U2, s2, _ = mat.computeSVD(k, True)
        torch.cuda.synchronize()
        out["gramian_jacobi_ms"] = round((time.perf_counter() - t) * 1e3, 1)
        out["max_s_diff_rel"] = float(np.abs(s - s2[:len(s)]).max() / s2[0])
        del U2
    print(json.dumps(out), flush=True)
    del U, mat, blk, buf
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--skip-svd", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eigs needs a CUDA device")
    mb.Runtime.get()
    gpu = card()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for m, n in [(1048576, 1024), (4194304, 256), (16384, 131072)]:
        bench_kernel(m, n, args, gpu, sms)
    if args.skip_svd:
        return
    bench_svd(1048576, 1024, 10, args, gpu)
    bench_svd(131072, 4096, 10, args, gpu, old=False)        # the Gramian and Jacobi path takes seconds here
    bench_svd(20000, 100000, 10, args, gpu, old=False)       # beyond that path's 65535-column cap


if __name__ == "__main__":
    main()

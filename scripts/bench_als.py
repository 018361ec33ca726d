"""CoordinateMatrix.ALS timings on one GPU: a MovieLens-20M-shaped problem (138493 x 26744, 20M ratings, power-law
activity) at ranks 10, 50 and 100, one explicit iteration, warm-up then best of 3 with CUDA events:
  - the whole iteration (mb_als_train), each half-step (mb_als_update), the assembly alone (mb_als_normal_equations)
    and the solve as the difference;
  - the host links build (mb_als_links, both sides);
  - rates from the shapes: assembly terms sum_u n_u r (r + 1) / 2, one DMUL and one DADD each, against the CUDA-core fp64
    issue rate (SMs x 64 lanes x SM clock, the DMUL / DADD rate, not a DFMA's two flops); solve flops n r^3 / 3; gather
    bytes nnz r 8;
  - the card name, power limit and SM clock, read in the same run;
  - a MovieLens-100K-shaped run (943 x 1682, 100k ratings) against the step-by-step oracle, for parity and context.
Prints one JSON line per measurement."""
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import marlin_b200 as mb  # noqa: E402
from marlin_b200 import _native as nat  # noqa: E402
from marlin_b200.matrix.coordinate_matrix import _Links  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()[0]
    name, power, sm, smmax = [s.strip() for s in q.split(",")]
    return {"card": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": smmax}


def shape(nu, ni, nnz, seed, a_u=0.6, a_i=0.9):
    rng = np.random.default_rng(seed)
    pu = 1.0 / np.arange(1, nu + 1) ** a_u
    pi = 1.0 / np.arange(1, ni + 1) ** a_i
    rows = rng.permutation(nu)[rng.choice(nu, nnz, p=pu / pu.sum())]
    cols = rng.permutation(ni)[rng.choice(ni, nnz, p=pi / pi.sum())]
    return rows, cols, (rng.integers(1, 11, nnz) / 2.0).astype(np.float32)


def timed(rt, fn, reps=3):
    fn()                                                   # warm-up
    best = float("inf")
    for _ in range(reps):
        nat.check(rt.lib.mb_timer_start(rt.ctx))
        fn()
        ms = C.c_float()
        nat.check(rt.lib.mb_timer_stop(rt.ctx, C.byref(ms)))
        best = min(best, ms.value)
    return best


def main():
    rt = mb.Runtime.get()
    rt.sync_stream()
    info = card()
    clock_hz = float(info["sm_clock"].split()[0]) * 1e6
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    issue = sms * 64 * clock_hz                            # fp64 CUDA-core instructions per second
    rows, cols, vals = shape(138493, 26744, 20_000_000, 2024)
    t0 = time.perf_counter()
    users = _Links(rows, cols, vals, 10, 10)
    products = _Links(cols, rows, vals, 10, 10)
    links_s = time.perf_counter() - t0
    print(json.dumps({"shape": "ml-20m", "links_host_s": round(links_s, 3), **info}), flush=True)
    us, keep_u = users.to_device(rt.device)
    ps, keep_p = products.to_device(rt.device)
    nnz = len(rows)
    for rank in (10, 50, 100):
        U = torch.rand(users.n * rank, dtype=torch.float64, device=rt.device)
        P = torch.rand(products.n * rank, dtype=torch.float64, device=rt.device)
        Ub = mb.SubMatrix(buf=U, rows=users.n, cols=rank, ld=rank, is_transpose=True)
        Pb = mb.SubMatrix(buf=P, rows=products.n, cols=rank, ld=rank, is_transpose=True)
        tri = rank * (rank + 1) // 2
        iter_ms = timed(rt, lambda: nat.check(rt.lib.mb_als_train(rt.ctx, C.byref(us), C.byref(ps), 1, 0.05, 1.0, 0,
                                                                  Ub.handle(), Pb.handle())))
        half = {}
        asm = {}
        for name, side, Y, X, L in (("products", ps, Ub, Pb, products), ("users", us, Pb, Ub, users)):
            half[name] = timed(rt, lambda: nat.check(rt.lib.mb_als_update(rt.ctx, C.byref(side), Y.handle(), 0.05, 1.0, 0,
                                                                          None, X.handle())))
            A = torch.empty(L.n * tri, dtype=torch.float64, device=rt.device)
            b = torch.empty(L.n * rank, dtype=torch.float64, device=rt.device)
            asm[name] = timed(rt, lambda: nat.check(rt.lib.mb_als_normal_equations(
                rt.ctx, C.byref(side), Y.handle(), 0.05, 1.0, 0, None, C.c_void_p(A.data_ptr()), C.c_void_p(b.data_ptr()))))
            del A, b
        terms = 2 * nnz * tri                             # both half-steps: every rating is a term on each side
        asm_ms = asm["products"] + asm["users"]
        print(json.dumps({
            "shape": "ml-20m", "rank": rank, "iteration_ms": round(iter_ms, 3),
            "half_step_ms": {k: round(v, 3) for k, v in half.items()},
            "assembly_ms": {k: round(v, 3) for k, v in asm.items()},
            "assembly_share_of_dmul_dadd_issue": round(2 * terms / (asm_ms * 1e-3) / issue, 4),
            "solve_ms": {k: round(half[k] - asm[k], 3) for k in half},   # half-step minus its assembly
            "solve_gflop_per_iteration": round((users.n + products.n) * rank ** 3 / 3 / 1e9, 3),
            "solve_gflop_s": round((users.n + products.n) * rank ** 3 / 3 / 1e9
                                   / max(1e-9, (half["users"] - asm["users"] + half["products"] - asm["products"]) * 1e-3), 1),
            "gather_gb_per_iteration": round(2 * nnz * rank * 8 / 1e9, 3),
            "gather_gb_s": round(2 * nnz * rank * 8 / (iter_ms * 1e-3) / 1e9, 1),
            **info}), flush=True)
        del U, P, Ub, Pb
    # MovieLens-100K shape against the oracle
    sys.path.insert(0, str(ROOT / "tests"))
    import als_oracle as ao
    rows, cols, vals = shape(943, 1682, 100_000, 7, 0.5, 0.8)
    for rank in (10, 50):
        t0 = time.perf_counter()
        Uf, Pf = mb.CoordinateMatrix((rows, cols, vals)).ALS(rank, 5, 0.05, 10, 10, seed=1)
        torch.cuda.synchronize()
        gpu_s = time.perf_counter() - t0
        t0 = time.perf_counter()
        _, U0, _, P0 = ao.als(rows, cols, vals, rank, 5, 0.05, 10, 10, seed=1)
        oracle_s = time.perf_counter() - t0
        U, P = Uf.data.toBreeze(), Pf.data.toBreeze()
        rel = max(np.abs(U - U0).max() / np.abs(U0).max(), np.abs(P - P0).max() / np.abs(P0).max())
        print(json.dumps({"shape": "ml-100k", "rank": rank, "iterations": 5, "gpu_s_end_to_end": round(gpu_s, 3),
                          "oracle_s": round(oracle_s, 2), "max_rel_diff_vs_oracle": float(rel), **info}), flush=True)


if __name__ == "__main__":
    main()

"""SparseVecMatrix.multiplySparse timings on one GPU (mb_spvec_multiply, the row-wise float32 SpGEMM):
  (a) the SparseMultiply example's mode-1 shapes, 16384 x 16384 times 16384 x 16384 from randomSpaVecMatrix at densities
      1e-3 and 1e-2 (every row of a partition shares its columns, so a row's products pile onto few columns), with the
      mode-2 dense multiply of the same matrices beside them;
  (b) a seeded R-MAT graph (scale 15, edge factor 16, a = 0.57, b = c = 0.19) squared, whose row product counts span all
      three bins (scale 18 squared has 2.9e9 products and more output entries than an int32 row pointer holds);
  (c) rows with independent uniform columns (262144 x 262144, 16 per row), squared.
For each: CUDA-event time of the whole call (best of 3 after a warm-up; the call includes its two host synchronisations),
the numeric pass alone (sum of the numeric kernels' durations in a separate torch.profiler run), products (sum over rows
of the B rows reached) per second, output nnz, the row counts per bin, and torch.sparse.mm on float32 CSR (cuSPARSE) as a
yardstick: same pattern, values within float tolerance (its summation order differs).  The card name and power limit are
read in the same run.  Prints one JSON line per measurement."""
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()[0]
    name, power, smmax = [s.strip() for s in q.split(",")]
    return {"card": name, "power_limit": power, "sm_clock_max": smmax}


def rmat(scale, edge_factor, seed, a=0.57, b=0.19, c=0.19):
    rng = np.random.default_rng(seed)
    n, m = 1 << scale, edge_factor << scale
    r = np.zeros(m, np.int64)
    col = np.zeros(m, np.int64)
    for bit in range(scale):
        u = rng.random(m)
        down = u >= a + b                     # quadrants c and d set the row bit
        right = ((u >= a) & (u < a + b)) | (u >= a + b + c)
        r |= down.astype(np.int64) << bit
        col |= right.astype(np.int64) << bit
    perm = rng.permutation(n)
    return n, perm[r], perm[col], rng.standard_normal(m)


def csr_matrix(n_rows, n_cols, r, c, v):
    key = np.unique(r * n_cols + c, return_index=True)[1]
    r, c, v = r[key], c[key], v[key]
    order = np.lexsort((c, r))
    r, c, v = r[order], c[order], v[order]
    rowptr = np.zeros(n_rows + 1, np.int64)
    np.add.at(rowptr, r + 1, 1)
    return mb.SparseVecMatrix((np.arange(n_rows), np.cumsum(rowptr), c, v), n_rows, n_cols)


def uniform_rows(n, per_row, seed):
    rng = np.random.default_rng(seed)
    r = np.repeat(np.arange(n), per_row)
    return csr_matrix(n, n, r, rng.integers(0, n, n * per_row), rng.standard_normal(n * per_row))


def run(rt, A, Bfull):
    out = nat.c_sp()
    nat.check(rt.lib.mb_spvec_multiply(rt.ctx, A.block.handle(), Bfull.handle(), C.byref(out)))
    return out


def measure(name, A, B, rt):
    Bfull = B._all_rows_csr()
    rt.sync_stream()
    rp_a, ci_a, _ = (t.cpu().numpy() for t in (A.block.colptr, A.block.rowidx, A.block.values))
    blen = np.diff(Bfull.colptr.cpu().numpy().astype(np.int64))
    per_row = np.add.reduceat(np.concatenate([blen[ci_a], [0]]), rp_a[:-1]) * (np.diff(rp_a) > 0)
    products = int(per_row.sum())
    bins = [int(((per_row > 0) & (per_row <= nat.MB_SPVEC_WARP_BOUND)).sum()),
            int(((per_row > nat.MB_SPVEC_WARP_BOUND) & (per_row <= nat.MB_SPVEC_CTA_BOUND)).sum()),
            int((per_row > nat.MB_SPVEC_CTA_BOUND).sum())]
    rt.lib.mb_sparse_free(rt.ctx, run(rt, A, Bfull))          # warm-up
    best = float("inf")
    for _ in range(3):
        nat.check(rt.lib.mb_timer_start(rt.ctx))
        h = run(rt, A, Bfull)
        ms = C.c_float()
        nat.check(rt.lib.mb_timer_stop(rt.ctx, C.byref(ms)))
        best = min(best, ms.value)
        nnz = nat.c_i64()
        nat.check(rt.lib.mb_sparse_info(h, None, None, C.byref(nnz)))
        rt.lib.mb_sparse_free(rt.ctx, h)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        rt.lib.mb_sparse_free(rt.ctx, run(rt, A, Bfull))
        torch.cuda.synchronize()
    numeric_us = sum(e.device_time_total for e in prof.key_averages() if "spvec" in e.key and "<true>" in e.key)
    # cuSPARSE yardstick on float32 CSR
    ta = torch.sparse_csr_tensor(A.block.colptr.long(), A.block.rowidx.long(), A.block.values.float(),
                                 size=(len(A.ids), A.nCols))
    tb = torch.sparse_csr_tensor(Bfull.colptr.long(), Bfull.rowidx.long(), Bfull.values.float(), size=(B.nRows, B.nCols))
    torch.sparse.mm(ta, tb)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    tc = torch.sparse.mm(ta, tb)
    torch.cuda.synchronize()
    cus_ms = (time.perf_counter() - t0) * 1e3
    ours = A.multiplySparse(B)
    o = np.lexsort((ours.cols, ours.rows))
    tcc = tc.to_sparse_coo().coalesce()
    idx = tcc.indices().cpu().numpy()
    same_pattern = idx.shape[1] == len(ours.rows) and np.array_equal(idx[0], ours.rows[o]) and np.array_equal(idx[1], ours.cols[o])
    diff = np.abs(tcc.values().cpu().numpy() - ours.values[o]) if same_pattern else np.zeros(1)
    close = bool(same_pattern and np.allclose(tcc.values().cpu().numpy(), ours.values[o], rtol=1e-4, atol=1e-5))
    rec = {"workload": name, "rows": len(A.ids), "a_nnz": A.block.nnz, "b_nnz": Bfull.nnz, "products": products,
           "out_nnz": int(nnz.value), "bins": bins, "call_ms": round(best, 3), "numeric_ms": round(numeric_us / 1e3, 3),
           "gproducts_per_s": round(products / best / 1e6, 3), "cusparse_ms": round(cus_ms, 3),
           "cusparse_same_pattern": bool(same_pattern), "cusparse_close": close,
           "cusparse_max_abs_diff": float(diff.max()) if diff.size else 0.0}
    print(json.dumps(rec), flush=True)
    return rec


def main():
    rt = mb.Runtime.get()
    print(json.dumps(card()), flush=True)
    for density in (1e-3, 1e-2):
        A = mb.MTUtils.randomSpaVecMatrix(None, 16384, 16384, density, seed=7)
        B = mb.MTUtils.randomSpaVecMatrix(None, 16384, 16384, density, seed=8)
        measure(f"mode1_16384_d{density:g}", A, B, rt)
        denA, denB = A.toDenseVecMatrix(), B.toDenseVecMatrix()
        torch.cuda.synchronize()
        denA.multiply(denB, (6, 6, 6))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        denA.multiply(denB, (6, 6, 6))
        torch.cuda.synchronize()
        print(json.dumps({"workload": f"mode2_16384_d{density:g}", "dense_multiply_ms": round((time.perf_counter() - t0) * 1e3, 3)}),
              flush=True)
        del denA, denB
    n, r, c, v = rmat(15, 16, seed=1)
    G = csr_matrix(n, n, r, c, v)
    measure("rmat_s15_ef16_squared", G, G, rt)
    U = uniform_rows(262144, 16, seed=2)
    measure("uniform_262144_16_squared", U, U, rt)


if __name__ == "__main__":
    main()

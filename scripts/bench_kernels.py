"""Secondary kernel benchmarks (1 GPU): HBM-bound block kernels vs the measured copy bandwidth, and the bf16 wgmma
GEMM vs cuBLAS, layout conversion, factorizations and the SVD.  Prints one JSON document; bench.py stays the headline
(fp64 multiply).  `svd` as an argument runs the f5_svd section only, `sparse` the f6_sparse section only."""
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import marlin_b200 as mb
from marlin_b200 import _native as nat

peaks = {}
try:
    peaks = json.loads((ROOT / "MEASURED_PEAKS.json").read_text())
except Exception:
    pass
HBM = float(peaks.get("hbm_gbs", 3350.0))
BF16 = float(peaks.get("bf16_tflops", 989.0))
rt = mb.Runtime.get()
out = {"hbm_peak_gbs": HBM, "bf16_peak_tflops": BF16, "peak_source": "MEASURED_PEAKS.json" if peaks else "fallback: H100 SXM data sheet, 700 W"}


def timeit(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


ONLY_SPARSE = "sparse" in sys.argv[1:]
ONLY_SVD = "svd" in sys.argv[1:]
SKIP_DENSE = ONLY_SVD or ONLY_SPARSE
hbm = {}
for n in (() if SKIP_DENSE else (8192, 16384)):
    A = mb.MTUtils.randomBlockMatrix(None, n, n, 1, 1, seed=1).blocks[0][1]
    B = mb.MTUtils.randomBlockMatrix(None, n, n, 1, 1, seed=2).blocks[0][1]
    O = mb.SubMatrix.empty(n, n)
    T = mb.SubMatrix.empty(n, n)
    lib, ctx = rt.lib, rt.ctx
    rt.sync_stream()
    elems = n * n
    cases = {
        "add (3*8 B/elem)": (lambda: nat.check(lib.mb_block_add(ctx, A.handle(), B.handle(), O.handle())), 24),
        "axpb (2*8 B/elem)": (lambda: nat.check(lib.mb_block_axpb(ctx, A.handle(), 2.0, 1.0, O.handle())), 16),
        "transpose (2*8 B/elem)": (lambda: nat.check(lib.mb_block_transpose(ctx, A.handle(), T.handle())), 16),
        "copy (2*8 B/elem)": (lambda: nat.check(lib.mb_block_copy(ctx, A.handle(), O.handle())), 16),
        "fill_uniform (8 B/elem)": (lambda: nat.check(lib.mb_fill_uniform(ctx, O.handle(), 7, 0, 0.0, 1.0, 0)), 8),
    }
    res = {}
    for name, (fn, bpe) in cases.items():
        ms = timeit(fn)
        gbs = elems * bpe / ms / 1e6
        res[name] = {"ms": ms, "GB/s": gbs, "frac_of_measured_hbm": gbs / HBM}
    # vector side (SURVEY 8f-4): the matrix crosses HBM once; vectors are noise
    xv, yv = mb.SubMatrix.empty(n, 1), mb.SubMatrix.empty(n, 1)
    nat.check(lib.mb_fill_uniform(ctx, xv.handle(), 3, 0, 0.0, 1.0, 0))
    At = A.t
    vec_cases = {
        "gemv y=A x (8 B/elem)": (lambda: nat.check(lib.mb_block_gemv(ctx, A.handle(), xv.handle(), yv.handle(), 0)), 8),
        "gemv y=A^T-view x, row-major rows (8 B/elem)": (lambda: nat.check(lib.mb_block_gemv(ctx, At.handle(), xv.handle(), yv.handle(), 0)), 8),
        "ger out=x y^T (8 B/elem written)": (lambda: nat.check(lib.mb_block_ger(ctx, xv.handle(), yv.handle(), O.handle())), 8),
    }
    for name, (fn, bpe) in vec_cases.items():
        ms = timeit(fn)
        gbs = elems * bpe / ms / 1e6
        res[name] = {"ms": ms, "GB/s": gbs, "frac_of_measured_hbm": gbs / HBM}
    s = C.c_double()
    Aflat = mb.SubMatrix(buf=A.buf, rows=elems, cols=1, ld=elems)
    Bflat = mb.SubMatrix(buf=B.buf, rows=elems, cols=1, ld=elems)
    ms = timeit(lambda: nat.check(lib.mb_block_dot(ctx, Aflat.handle(), Bflat.handle(), C.byref(s))))
    res["dot (2*8 B/elem, incl. D2H of the scalar)"] = {"ms": ms, "GB/s": elems * 16 / ms / 1e6, "frac_of_measured_hbm": elems * 16 / ms / 1e6 / HBM}
    ms = timeit(lambda: nat.check(lib.mb_block_sum(ctx, A.handle(), C.byref(s))))
    res["sum (8 B/elem, incl. D2H of the scalar)"] = {"ms": ms, "GB/s": elems * 8 / ms / 1e6, "frac_of_measured_hbm": elems * 8 / ms / 1e6 / HBM}
    ta = torch.empty(elems, dtype=torch.float64, device="cuda")
    tb = torch.empty(elems, dtype=torch.float64, device="cuda")
    ms = timeit(lambda: tb.copy_(ta))
    res["torch copy_ yardstick (2*8 B/elem)"] = {"ms": ms, "GB/s": elems * 16 / ms / 1e6}
    hbm[f"{n}x{n} fp64"] = res
    del A, B, O, T, ta, tb, At, Aflat, Bflat
out["hbm_kernels"] = hbm

gemm = {}
for n in (() if SKIP_DENSE or "hbm" in sys.argv[1:] else (4096, 8192, 16384)):
    A = mb.MTUtils.randomBlockMatrix(None, n, n, 1, 1, seed=3, dtype=nat.MB_BF16).blocks[0][1]
    B = mb.MTUtils.randomBlockMatrix(None, n, n, 1, 1, seed=4, dtype=nat.MB_BF16).blocks[0][1]
    Cm = mb.SubMatrix.empty(n, n, nat.MB_F32)
    C16 = mb.SubMatrix.empty(n, n, nat.MB_BF16)
    iters = 10 if n <= 8192 else 4
    ms32 = timeit(lambda: A.multiply(B, out=Cm), iters)
    ms16 = timeit(lambda: A.multiply(B, out=C16), iters)
    ta = A.buf.view(n, n)
    tb = B.buf.view(n, n)
    tc = torch.empty(n, n, dtype=torch.bfloat16, device="cuda")
    msc = timeit(lambda: torch.matmul(tb, ta, out=tc), iters)        # column-major A*B == row-major B^T... same flops
    fl = 2.0 * n ** 3
    gemm[f"{n}^3"] = {"ours_f32out_ms": ms32, "ours_f32out_tflops": fl / ms32 / 1e9, "ours_bf16out_ms": ms16,
                      "ours_bf16out_tflops": fl / ms16 / 1e9, "cublas_bf16_ms": msc, "cublas_bf16_tflops": fl / msc / 1e9,
                      "frac_of_measured_bf16_peak": fl / ms32 / 1e9 / BF16}
    del A, B, Cm, C16, ta, tb, tc
out["bf16_gemm"] = gemm

# ---- f1: layout conversion on the device (rows -> blocks -> rows), 2 * 8 * M * N bytes per direction ----
f1 = {}
for (M_, N_, gr, gc) in (() if SKIP_DENSE or "hbm" in sys.argv[1:] else ((16384, 16384, 2, 2), (1048576, 1024, 8, 1))):
    D = mb.MTUtils.randomDenVecMatrix(None, M_, N_, numPartitions=1, seed=5)
    torch.cuda.synchronize()
    Bm = D.toBlockMatrix(gr, gc)
    ms_rb = timeit(lambda: D.toBlockMatrix(gr, gc), 5, 2)
    ms_br = timeit(lambda: Bm.toDenseVecMatrix(), 5, 2)
    ms_rg = timeit(lambda: Bm.toBlockMatrix(gr * 2, gc), 5, 2)
    by = 16.0 * M_ * N_
    f1[f"{M_}x{N_} fp64, {gr}x{gc} grid"] = {
        "rows_to_blocks": {"ms": ms_rb, "GB/s": by / ms_rb / 1e6, "frac_of_measured_hbm": by / ms_rb / 1e6 / HBM},
        "blocks_to_rows": {"ms": ms_br, "GB/s": by / ms_br / 1e6, "frac_of_measured_hbm": by / ms_br / 1e6 / HBM},
        "regrid": {"ms": ms_rg, "GB/s": by / ms_rg / 1e6, "frac_of_measured_hbm": by / ms_rg / 1e6 / HBM}}
    del D, Bm
    torch.cuda.empty_cache()
out["f1_layout_conversion"] = f1

# ---- f4: factorizations of one block (recursive; the flops run in the DMMA GEMM) ----
fac = {}
for n in (() if SKIP_DENSE or "hbm" in sys.argv[1:] else (4096, 8192)):
    A = mb.MTUtils.randomBlockMatrix(None, n, n, 1, 1, seed=6).blocks[0][1]
    S = A.multiply(A.t)
    S.add_(mb.SubMatrix(torch.eye(n, dtype=torch.float64).mul_(float(n)).numpy(), device=rt.device))
    ms_lu = timeit(lambda: A.lu(), 3, 1)
    ms_ch = timeit(lambda: S.cholesky(), 3, 1)
    ms_inv = timeit(lambda: S.inverse(), 3, 1)
    fac[f"{n}^2"] = {"lu_ms": ms_lu, "lu_tflops": (2.0 / 3.0) * n ** 3 / ms_lu / 1e9, "cholesky_ms": ms_ch,
                     "cholesky_tflops": (1.0 / 3.0) * n ** 3 / ms_ch / 1e9, "inverse_ms": ms_inv, "inverse_tflops": 2.0 * n ** 3 / ms_inv / 1e9,
                     "note": "times include the working copy of the block and, for LU, the D2H of the pivots"}
    del A, S
out["f4_factorizations"] = fac

# ---- f5: DenseVecMatrix.computeSVD — split-K DMMA Gramian, Jacobi eigensolver, end to end ----
f5 = {}
if "hbm" not in sys.argv[1:] and not ONLY_SPARSE:
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                          str(rt.device_index)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    f5["device"] = {"torch_name": torch.cuda.get_device_name(rt.device_index), "nvidia_smi": smi.stdout.strip()}
    gram = {}
    for (M_, N_) in ((1048576, 1024), (131072, 4096)):
        D = mb.MTUtils.randomDenVecMatrix(None, M_, N_, numPartitions=1, seed=8)
        X = D.data                                   # the row shard: a transposed view, read in place
        full = mb.SubMatrix.empty(N_, N_)
        ms_g = timeit(lambda: X.gramian(), 5, 2)
        ms_f = timeit(lambda: X.t.multiply(X, out=full), 5, 2)
        fl_g, fl_f = float(M_) * N_ * (N_ + 1), 2.0 * M_ * N_ * N_
        gram[f"{M_}x{N_}"] = {"gramian_ms": ms_g, "gramian_tflops_mn(n+1)": fl_g / ms_g / 1e9,
                              "full_gemm_AtA_ms": ms_f, "full_gemm_tflops_2mn^2": fl_f / ms_f / 1e9}
        del D, X, full
        torch.cuda.empty_cache()
    f5["gramian"] = gram
    eig = {}
    for n in (256, 1024, 4096):
        rng_rows = mb.MTUtils.randomDenVecMatrix(None, 2 * n, n, numPartitions=1, seed=9)
        G = rng_rows.data.gramian()
        G.symmetricEigen()                           # warm-up (module load)
        torch.cuda.synchronize()
        reps = 3 if n <= 1024 else 1
        t0 = time.perf_counter()
        for _ in range(reps):
            w, V = G.symmetricEigen()
        ms = (time.perf_counter() - t0) * 1e3 / reps
        eig[f"n={n}"] = {"ms": ms, "sweeps": G.last_sweeps, "ms_per_sweep": ms / max(1, G.last_sweeps),
                         "note": "host clock around the blocking call: copies, N-1 rounds per sweep, ordering, gather"}
        del rng_rows, G, V
        torch.cuda.empty_cache()
    f5["eigensolver"] = eig
    # where a sweep's time goes: the round kernels' device time vs the gaps between consecutive rounds of a graph replay
    # (the launch overhead a persistent grid-barrier kernel could replace with a barrier), and the per-call set-up
    # (working copies, graph capture and instantiation, ordering, gather) as wall time minus the device span
    from torch.profiler import ProfilerActivity, profile
    prof_out = {}
    for n in (256, 1024):
        rows_ = mb.MTUtils.randomDenVecMatrix(None, 2 * n, n, numPartitions=1, seed=9)
        G = rows_.data.gramian()
        G.symmetricEigen()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            t0 = time.perf_counter()
            G.symmetricEigen()
            wall = (time.perf_counter() - t0) * 1e3
        evs = sorted([e for e in prof.events() if "jacobi_" in e.name and e.device_type.name == "CUDA"],
                     key=lambda e: e.time_range.start)
        rounds = [e for e in evs if "jacobi_round_kernel" in e.name]
        if len(rounds) < 2:
            prof_out[f"n={n}"] = {"wall_ms": wall, "note": "round kernels not captured by the profiler"}
            continue
        dur = sorted(e.time_range.elapsed_us() for e in rounds)
        gaps = sorted(b.time_range.start - a.time_range.end for a, b in zip(rounds, rounds[1:]))
        span_ms = (evs[-1].time_range.end - evs[0].time_range.start) / 1e3
        prof_out[f"n={n}"] = {"rounds": len(rounds), "sweeps": G.last_sweeps, "round_kernel_us_median": dur[len(dur) // 2],
                              "gap_between_rounds_us_median": gaps[len(gaps) // 2],
                              "round_kernels_ms_total": sum(dur) / 1e3, "device_span_ms": span_ms, "wall_ms": wall,
                              "setup_and_host_ms": wall - span_ms}
        del rows_, G
    f5["eigensolver_breakdown"] = prof_out
    D = mb.MTUtils.randomDenVecMatrix(None, 1048576, 1024, numPartitions=1, seed=10)
    D.computeSVD(10, computeU=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    U, s_, V_ = D.computeSVD(10, computeU=True)
    torch.cuda.synchronize()
    f5["computeSVD_k10_U_1048576x1024_ms"] = (time.perf_counter() - t0) * 1e3
    del D, U
    torch.cuda.empty_cache()
out["f5_svd"] = f5


# ---- f6: sparse blocks — the three sparse products against DMMA on the same block made dense, the generator, and
#      BlockMatrix.multiply in the reference's SparseMultiply modes.  The sparse kernels sum in the reference's order with
#      separate multiplies and adds, so they are bound by memory traffic, not by the tensor cores. ----
def timed(fn, budget_ms=1500.0):
    """Mean ms per call: one warm-up call, then as many calls as fit in about budget_ms (at least one, at most 10)."""
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    first = (time.perf_counter() - t0) * 1e3
    iters = int(max(1, min(10, budget_ms / max(first, 1e-3))))
    return timeit(fn, iters, 0) if iters > 1 else first


f6 = {}
if ONLY_SPARSE or not (ONLY_SVD or "hbm" in sys.argv[1:]):
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                          str(rt.device_index)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    f6["device"] = {"torch_name": torch.cuda.get_device_name(rt.device_index), "nvidia_smi": smi.stdout.strip()}
    densities = (1e-4, 1e-3, 1e-2, 5e-2, 0.1)
    kernels = {}
    for n in (4096, 16384):
        D = mb.MTUtils.randomBlockMatrix(None, n, n, 1, 1, seed=21).blocks[0][1]
        O = mb.SubMatrix.empty(n, n)
        ms_dmma = timed(lambda: D.multiply(D, out=O))
        per_n = {"dmma_dense_product_ms": ms_dmma, "by_density": {}}
        for d in densities:
            S = mb.MTUtils.randomBlockMatrix(None, n, n, 1, 1, (True, d), seed=22).blocks[0][1]
            nnz = S.sparseBlock.nnz
            s = nnz // n
            sp_bytes = 12.0 * nnz
            dense_io = 16.0 * n * n                                  # read the dense operand once, write C once
            row = {"nnz": nnz}
            for name, fn, flops, by in (
                    ("dense_x_sparse", lambda: D.multiply(S, out=O), 2.0 * n * nnz, dense_io + sp_bytes),
                    ("sparse_x_dense", lambda: S.multiply(D, out=O), 2.0 * n * nnz, dense_io + sp_bytes),
                    ("sparse_x_sparse", lambda: S.multiply(S, out=O), 2.0 * nnz * s, 8.0 * n * n + 2 * sp_bytes)):
                # the first call on a fresh block: for sparse x dense it includes building the cached CSR copy
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                first_ms = (time.perf_counter() - t0) * 1e3
                ms = timed(fn)
                row[name] = {"ms": ms, "gflops": flops / ms / 1e6, "min_bytes": by, "GB/s_of_min_bytes": by / ms / 1e6,
                             "speedup_vs_dmma": ms_dmma / ms, "first_call_ms": first_ms}
            per_n["by_density"][str(d)] = row
            del S
            torch.cuda.empty_cache()
        # crossover: the densities bracketing the point where the sparse kernel stops beating DMMA on the dense block
        cross = {}
        for name in ("dense_x_sparse", "sparse_x_dense", "sparse_x_sparse"):
            for key, label in (("ms", ""), ("first_call_ms", "_first_call")):
                wins = [d for d in densities if per_n["by_density"][str(d)][name][key] < ms_dmma]
                loses = [d for d in densities if per_n["by_density"][str(d)][name][key] >= ms_dmma]
                cross[name + label] = {"sparse_wins_up_to": max(wins) if wins else None,
                                       "dmma_wins_from": min(loses) if loses else None}
        per_n["crossover_density"] = cross
        kernels[f"{n}^2"] = per_n
        del D, O
        torch.cuda.empty_cache()
    f6["kernels"] = kernels
    n = 16384
    ms_gen = timed(lambda: mb.MTUtils.randomBlockMatrix(None, n, n, 1, 1, (True, 1e-3), seed=23))
    ms_fill = timed(lambda: mb.MTUtils.randomBlockMatrix(None, n, n, 1, 1, seed=23))
    f6["generator_16384^2"] = {"sparse_density_1e-3_ms": ms_gen, "dense_fill_ms": ms_fill,
                               "note": "the sparse generator draws rows*cols stream positions whatever the density"}
    modes = {}
    d = 1e-3
    Ad = mb.MTUtils.randomBlockMatrix(None, n, n, 2, 2, seed=24)
    As = mb.MTUtils.randomBlockMatrix(None, n, n, 2, 2, (True, d), seed=25)
    Bs = mb.MTUtils.randomBlockMatrix(None, n, n, 2, 2, (True, d), seed=26)
    Asd, Bsd = As.toDenseBlocks(), Bs.toDenseBlocks()           # converted before the clock starts, as in the reference
    for mode, fn in (("3_sparse_x_sparse", lambda: As.multiply(Bs)),
                     ("4_dense_blocks_x_dense_blocks", lambda: Asd.multiply(Bsd)),
                     ("5_dense_x_sparse", lambda: Ad.multiply(Bs)),
                     ("6_dense_x_sparse_as_dense_blocks", lambda: Ad.multiply(Bsd))):
        modes[mode] = {"ms": timed(lambda: (fn(), torch.cuda.synchronize()))}
        torch.cuda.empty_cache()
    f6[f"SparseMultiply_16384^2_2x2_density_{d}"] = modes
    del Ad, As, Bs, Asd, Bsd
    torch.cuda.empty_cache()
out["f6_sparse"] = f6
Path("gpurun_out").mkdir(exist_ok=True)
Path("gpurun_out/kernels.json").write_text(json.dumps(out, indent=1))
print(json.dumps(out, indent=1))

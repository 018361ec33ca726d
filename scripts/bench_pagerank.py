"""PageRank iteration timings on one GPU (mb_pagerank_step over the in-link CSR, the example's numBlocks = 2 segments):
  (a) a uniform random graph of 2^22 pages with 16 in-links per page on average;
  (b) a seeded R-MAT graph, scale 22 and edge factor 16 (a = 0.57, b = c = 0.19), whose in-degrees are heavy-tailed;
  (c) a star: one page with 2^20 - 1 in-links inside 2^20 pages, which shows the cost of one row's serial chain;
  (d) the graphs of (a) and (b) at 16384 and 32768 pages, beside the dense composition of the library's public
      operations (loadLinksMatrix(...).toDenseVecMatrix().transpose(2).multiply(0.85), then links.multiply(ranks), the
      reduce, + 0.15 and the re-split per iteration), which reads the whole n x n link matrix every iteration.
For each: CUDA-event time per iteration (a warm-up, then the best of 3 runs of 10 steps), the setup time apart (the host
in-link build, and the upload with the one-time binning), and the compulsory bytes per iteration (12 * nnz for sources and
weights, 12 * n for the row pointers and y) with the x gathers (8 * nnz at most) listed apart, over the time.  The card
name and power limit are read in the same run.  Prints one JSON line per measurement."""
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
from marlin_b200.examples import page_rank as pr  # noqa: E402
from marlin_b200.matrix.sub_matrix import SubMatrix  # noqa: E402
from tests import pagerank_oracle as po  # noqa: E402

STEPS = 10


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()[0]
    name, power, smmax = [s.strip() for s in q.split(",")]
    return {"card": name, "power_limit": power, "sm_clock_max": smmax}


def uniform(n, per_page, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(0, n, n * per_page), rng.integers(0, n, n * per_page)


def star(n):
    return np.concatenate([np.arange(1, n), [0]]), np.concatenate([np.zeros(n - 1, np.int64), [n - 1]])


def measure(name, n, src, dst, rt):
    rows = po.link_rows(src, dst, n)
    m = mb.SparseVecMatrix(rows, n, n)
    parts = m._gathered()
    t1 = time.perf_counter()
    links = pr._in_links(parts, n, 0, n)
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    seg = (n + 1) // 2
    x = torch.ones(n, dtype=torch.float64, device=rt.device)
    y = torch.empty_like(x)
    xv, yv = SubMatrix(buf=x, rows=n, cols=1, ld=n), SubMatrix(buf=y, rows=n, cols=1, ld=n)
    rt.sync_stream()
    t3 = time.perf_counter()
    nat.check(rt.lib.mb_pagerank_step(rt.ctx, links.handle(), xv.handle(), seg, pr.TELEPORT, yv.handle()))   # bins once
    torch.cuda.synchronize()
    bin_s = time.perf_counter() - t3
    best = float("inf")
    for _ in range(3):
        nat.check(rt.lib.mb_timer_start(rt.ctx))
        for _ in range(STEPS):
            nat.check(rt.lib.mb_pagerank_step(rt.ctx, links.handle(), xv.handle(), seg, pr.TELEPORT, yv.handle()))
        ms = C.c_float()
        nat.check(rt.lib.mb_timer_stop(rt.ctx, C.byref(ms)))
        best = min(best, ms.value / STEPS)
    deg = np.bincount(np.asarray(rows[2]), minlength=n)
    nnz = links.nnz
    compulsory = 12 * nnz + 12 * n
    rec = {"workload": name, "pages": n, "in_links": int(nnz), "max_in_degree": int(deg.max()),
           "heavy_rows": int((deg > nat.MB_PAGERANK_LIGHT_BOUND).sum()), "iteration_ms": round(best, 4),
           "setup_links_s": round(t2 - t1, 3), "setup_bin_s": round(bin_s, 3), "compulsory_bytes": int(compulsory),
           "gather_bytes_max": int(8 * nnz), "compulsory_gb_per_s": round(compulsory / best / 1e6, 1)}
    print(json.dumps(rec), flush=True)
    return m


def measure_dense(name, m, n, rt):
    links = m.toDenseVecMatrix().transpose(2).multiply(0.85)
    ranks = mb.MTUtils.onesDistVector(None, n, 2)
    r = np.ones(n) * pr.TELEPORT

    def iteration(ranks):
        res = links.multiply(ranks)
        acc = None
        for _, v in sorted(res.getVectors, key=lambda t: t[0]):
            acc = v.toBreeze().reshape(-1) if acc is None else acc + v.toBreeze().reshape(-1)
        return mb.DistributedVector.fromVector(None, acc + r, 2)

    ranks = iteration(ranks)
    torch.cuda.synchronize()
    best = float("inf")
    for _ in range(3):
        t0 = time.perf_counter()
        ranks = iteration(ranks)
        torch.cuda.synchronize()
        best = min(best, time.perf_counter() - t0)
    print(json.dumps({"workload": name, "pages": n, "dense_iteration_ms": round(best * 1e3, 3),
                      "dense_link_bytes": 8 * n * n, "dense_gb_per_s": round(8 * n * n / best / 1e9, 1)}), flush=True)
    del links


def main():
    rt = mb.Runtime.get()
    print(json.dumps(card()), flush=True)
    measure("uniform_2^22_16", 1 << 22, *uniform(1 << 22, 16, seed=1), rt)
    measure("rmat_s22_ef16", 1 << 22, *po.rmat(22, 16, seed=2), rt)
    measure("star_2^20", 1 << 20, *star(1 << 20), rt)
    for n in (16384, 32768):
        m = measure(f"uniform_{n}_16", n, *uniform(n, 16, seed=3), rt)
        measure_dense(f"dense_uniform_{n}_16", m, n, rt)
        scale = n.bit_length() - 1
        m = measure(f"rmat_s{scale}_ef16", n, *po.rmat(scale, 16, seed=4), rt)
        measure_dense(f"dense_rmat_s{scale}_ef16", m, n, rt)


if __name__ == "__main__":
    main()

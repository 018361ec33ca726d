"""examples/PageRank.scala — `page_rank <file> [iteration=0] [linkNum=8]`: load a link file (`source target` per line,
pages 1-based) and iterate ranks = 0.85 * links^T * ranks + 0.15 over numBlocks = 2 pieces.

Deviations from the reference:
  - loadLinksMatrix returns the link rows as a SparseVecMatrix with the reference's values and row presence (its
    toDenseVecMatrix() is the reference's dense return value); the reference stores linkNum doubles per row.
  - The iteration runs on the in-link CSR of the link matrix (mb_pagerank_step / mb_pagerank_train), not on the dense
    blocks of linkRows.transpose(2).multiply(0.85).  Each rank's sum adds only the stored links, in ascending source order
    and split at the same block boundary, so the ranks are the dense reference's bit for bit (DESIGN §3.12).
  - A page id outside [1, linkNum] or an unparsable line raises MarlinArgumentError naming the line, where the reference
    fails with an index or number-format exception.
  - main prints the dense link rows only for linkNum <= 100 (they are O(linkNum^2) text) and otherwise one summary line;
    it prints the initial pieces' values where the reference prints an array's identity hash (DenseVector.toString).
"""
from __future__ import annotations

import ctypes as C
import math
import os
import re
import sys

import numpy as np
import torch

from .. import _native as nat
from .. import comm
from ..matrix.dense_vec_matrix import _ceil_len
from ..matrix.distributed_vector import DistributedVector
from ..matrix.sparse_matrix import SparseBlock
from ..matrix.sparse_vec_matrix import SparseVecMatrix
from ..matrix.sub_matrix import SubMatrix
from ..runtime import Runtime, world
from ..utils.mt_utils import MTUtils, _check_path, _jdouble

NUM_BLOCKS = 2          # numBlocks of the example
DAMPING = 0.85          # linkRows.transpose(numBlocks).multiply(0.85)
TELEPORT = 0.15         # BDV.ones(linkNum) * 0.15
DUMP_LIMIT = 100        # main prints the dense link rows up to this linkNum

_WS = re.compile(r"\s+")
_INT = re.compile(r"[+-]?[0-9]+")


def _page(token: str, line: str, what: str, linkNum: int) -> int:
    """parts(i).toLong / .toInt of one field, then the reference's array index range."""
    if not _INT.fullmatch(token):
        raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, f"PageRank: the {what} page of line {line!r} is not a number")
    v = int(token)
    if not 1 <= v <= linkNum:
        raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG,
                                      f"PageRank: the {what} page {v} of line {line!r} is outside [1, {linkNum}]")
    return v


def _parse(lines, linkNum: int):
    """(sources, targets) 0-based of `source target ...` lines split as String.split("\\\\s+") splits them."""
    src, dst = [], []
    for line in lines:
        parts = _WS.split(line)
        while parts and parts[-1] == "":            # java.lang.String.split drops trailing empty strings
            parts.pop()
        if len(parts) < 2:
            raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, f"PageRank: line {line!r} has no target page")
        src.append(_page(parts[0], line, "source", linkNum) - 1)
        dst.append(_page(parts[1], line, "target", linkNum) - 1)
    return np.array(src, np.int64), np.array(dst, np.int64)


def loadLinksMatrix(sc, input: str, linkNum: int) -> SparseVecMatrix:      # noqa: A002
    """PageRank.scala:13-27 — row `page - 1` of every page with out-links holds 1.0 / links.size at each of its targets,
    where links.size counts the page's lines (duplicates included) and a repeated target is stored once.  Lines are dealt
    to ranks in contiguous chunks as MTUtils.loadMatrixFile deals them; blank lines are skipped.  Row `page - 1` is held
    by rank (page - 1) mod G.  Every rank raises if any rank's lines hold an error."""
    linkNum = int(linkNum)
    if linkNum < 1:
        raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, f"PageRank: linkNum {linkNum} must be positive")
    _check_path(input)
    files = [input] if os.path.isfile(input) else sorted(os.path.join(input, f) for f in os.listdir(input)
                                                         if not f.startswith((".", "_")))
    lines = []
    for f in files:
        with open(f) as fh:
            lines.extend(l.rstrip("\r\n") for l in fh if l.strip())
    rank, ws = world()
    lo, hi = (rank * len(lines)) // ws, ((rank + 1) * len(lines)) // ws
    try:
        mine, err = _parse(lines[lo:hi], linkNum), None
    except nat.MarlinArgumentError as e:
        mine, err = None, str(e)
    if ws > 1:                                      # groupByKey: every rank sees every link, keeps its own pages
        import torch.distributed as dist
        everyone = [None] * ws
        dist.all_gather_object(everyone, (mine, err))
    else:
        everyone = [(mine, err)]
    errs = [e for _, e in everyone if e is not None]
    if errs:
        raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, errs[0])
    src = np.concatenate([m[0] for m, _ in everyone])
    dst = np.concatenate([m[1] for m, _ in everyone])
    keep = src % ws == rank
    src, dst = src[keep], dst[keep]
    ids, size = np.unique(src, return_counts=True)
    pairs = np.unique(src * linkNum + dst)            # (source, target) ascending, each once
    rows, cols = pairs // linkNum, pairs % linkNum
    per_row = np.searchsorted(rows, ids, side="right") - np.searchsorted(rows, ids, side="left")
    rowptr = np.concatenate([[0], np.cumsum(per_row)])
    vals = np.repeat(1.0 / size.astype(np.float64), per_row)
    return SparseVecMatrix((ids, rowptr, cols, vals), linkNum, linkNum)


def _in_links(parts, n: int, t0: int, t1: int) -> SparseBlock:
    """The in-link CSR of targets [t0, t1) from every rank's link rows (mb_pagerank_links), on this rank's device."""
    ids = np.ascontiguousarray(np.concatenate([p[0] for p in parts]), np.int64)
    lens = np.concatenate([np.diff(p[1]) for p in parts])
    rowptr = np.ascontiguousarray(np.concatenate([[0], np.cumsum(lens)]), np.int64)
    targets = np.ascontiguousarray(np.concatenate([p[2] for p in parts]), np.int32)
    values = np.ascontiguousarray(np.concatenate([p[3] for p in parts]), np.float64)
    nnz_cap = max(int(rowptr[-1]), 1)
    in_rp = np.empty(t1 - t0 + 1, np.int32)
    src = np.empty(nnz_cap, np.int32)
    w = np.empty(nnz_cap, np.float64)
    nnz = nat.c_i64()
    nat.check(nat.load().mb_pagerank_links(n, len(ids), ids.ctypes.data, rowptr.ctypes.data, targets.ctypes.data,
                                           values.ctypes.data, t0, t1, DAMPING, in_rp.ctypes.data, src.ctypes.data,
                                           w.ctypes.data, C.byref(nnz)))
    dev = Runtime.get().device
    k = int(nnz.value)
    return SparseBlock(n, t1 - t0, torch.from_numpy(in_rp).to(dev), torch.from_numpy(src[:k]).to(dev),
                       torch.from_numpy(w[:k]).to(dev))


def pageRank(linkRows: SparseVecMatrix, iterations: int) -> DistributedVector:
    """The loop of PageRank.scala:41-59 on the link rows of loadLinksMatrix: the final `ranks`, 2 pieces of
    ceil(n / 2) (the last takes the rest), piece i on rank i mod G.  iterations <= 0 gives the ones vector.  Where the dense
    composition linkRows.toDenseVecMatrix().transpose(2).multiply(0.85).multiply(ranks) raises (fewer than 4 pages), this
    raises the same error.

    One rank runs the whole loop on its GPU (mb_pagerank_train).  With several ranks every rank gathers the link rows,
    builds the in-links of the pieces it owns, and each iteration computes them (mb_pagerank_step) and exchanges them.  A
    row's arithmetic does not depend on which rank computes it, so the ranks are the same bits on any number of ranks."""
    n = int(linkRows.nRows)
    if linkRows.nCols != n or n < 1:
        raise nat.MarlinArgumentError(nat.MB_ERR_DIM_MISMATCH, f"PageRank: the link rows are {n} x {linkRows.nCols}, "
                                      "expected a square matrix of at least one page")
    iterations = int(iterations)
    if iterations <= 0:
        return MTUtils.onesDistVector(None, n, NUM_BLOCKS)
    # the block grid of transpose(2) as DenseVecMatrix.transpose computes it (n = 1 divides by n // 2 = 0 there), and
    # BlockMatrix.multiply(DistributedVector)'s check of it against the 2 pieces of ranks
    by_col = int(math.ceil(n / _ceil_len(n, min(NUM_BLOCKS, n // 2))))
    if by_col != NUM_BLOCKS:
        raise nat.MarlinArgumentError(nat.MB_ERR_UNSUPPORTED, "not supported matrix or vector")
    seg = _ceil_len(n, NUM_BLOCKS)
    bounds = [(0, seg), (seg, n)]
    rank, ws = world()
    parts = linkRows._gathered()
    rt = Runtime.get()
    if ws == 1:
        links = _in_links(parts, n, 0, n)
        x = SubMatrix.zeros(n, 1, nat.MB_F64).add(1.0)
        rt.sync_stream()
        nat.check(rt.lib.mb_pagerank_train(rt.ctx, links.handle(), seg, TELEPORT, iterations, x.handle()))
        return DistributedVector([(p, x.slice(t0, t1, 0, 1).copy()) for p, (t0, t1) in enumerate(bounds)], n, NUM_BLOCKS)
    import torch.distributed as dist
    owner = lambda p: p % ws                        # noqa: E731
    mine = [p for p in range(NUM_BLOCKS) if owner(p) == rank]
    links = {p: _in_links(parts, n, *bounds[p]) for p in mine}
    cpu = dist.get_backend() != "nccl"
    x = torch.ones(n, dtype=torch.float64, device=rt.device)
    sends = [(owner(p), dst, p) for p in range(NUM_BLOCKS) for dst in range(ws) if dst != owner(p)]
    for _ in range(iterations):
        out = {}
        for p in mine:
            t0, t1 = bounds[p]
            y = torch.empty(t1 - t0, dtype=torch.float64, device=rt.device)
            xv, yv = SubMatrix(buf=x, rows=n, cols=1, ld=n), SubMatrix(buf=y, rows=t1 - t0, cols=1, ld=max(1, t1 - t0))
            rt.sync_stream()                        # xv and yv are held: their handles must outlive the call
            nat.check(rt.lib.mb_pagerank_step(rt.ctx, links[p].handle(), xv.handle(), seg, TELEPORT, yv.handle()))
            out[p] = y
        local = {p: (y.cpu() if cpu else y) for p, y in out.items()}
        got = comm.exchange(sends, local, lambda p: torch.empty(bounds[p][1] - bounds[p][0], dtype=torch.float64,
                                                                device="cpu" if cpu else rt.device), rank)
        x = torch.cat([(out[p] if p in out else got[p].to(rt.device)) for p in range(NUM_BLOCKS)])
    return DistributedVector([(p, SubMatrix(buf=x[t0:t1].clone(), rows=t1 - t0, cols=1, ld=max(1, t1 - t0)))
                              for p, (t0, t1) in enumerate(bounds) if p in mine], n, NUM_BLOCKS)


def main(args):
    from ._common import start, stop
    if len(args) < 1:
        print("Usage: PageRank <file> <iteration> <linkNum>", file=sys.stderr)
        sys.exit(1)
    mb, rank = start()
    iteration = int(args[1]) if len(args) > 1 else 0
    linkNum = int(args[2]) if len(args) > 2 else 8
    linkRows = loadLinksMatrix(None, args[0], linkNum)
    parts = linkRows._gathered()
    if rank == 0:
        if linkNum <= DUMP_LIMIT:                   # linkRows.printAll()
            for ids, rp, ci, va in parts:
                for r, page in enumerate(ids):
                    row = np.zeros(linkNum)
                    row[ci[rp[r]:rp[r + 1]]] = va[rp[r]:rp[r + 1]]
                    print(f"index: {int(page)}, vector: " + ",".join(_jdouble(v) for v in row))
        else:
            print(f"{linkNum} pages, {sum(len(p[0]) for p in parts)} with out-links, "
                  f"{sum(len(p[2]) for p in parts)} stored links")
    ones = MTUtils.onesDistVector(None, linkNum, NUM_BLOCKS)
    pieces = ones._gather([(i, v.toBreeze().reshape(-1)) for i, v in ones.vectors])
    if rank == 0:                                   # ranks.getVectors.collect().foreach(println _)
        for i, v in sorted(pieces, key=lambda t: t[0]):
            print(f"({i}," + ",".join(_jdouble(a) for a in v) + ")")
        for i in range(iteration):
            print(f"in iteration {i}")
    final = pageRank(linkRows, iteration)
    final = final._gather([(i, v.toBreeze().reshape(-1)) for i, v in final.vectors])
    if rank == 0:
        for _, v in sorted(final, key=lambda t: t[0]):
            print("ranks: " + ", ".join(_jdouble(a) for a in v))
    stop()


if __name__ == "__main__":
    main(sys.argv[1:])

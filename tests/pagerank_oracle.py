"""CPU oracle of the PageRank example (examples/PageRank.scala).

`dense` runs the example literally on oracle/reference_model.py: the link rows as a DenseVecMatrix (only the pages with
out-links), transpose(2), multiply(0.85), then per iteration multiply_dist_vector (F2J dgemv per block), the reduce, the
add of 0.15 and the re-split into 2 pieces.  `InLinks.run` is the sparse sequential formulation the library computes:
per target, the products of its stored in-links in ascending source order summed from 0.0 per block column, the block
sums folded in order, then + 0.15.  It is vectorised in numpy by in-link position, so it reaches millions of edges.
"""
from __future__ import annotations

import math
import re

import numpy as np

NUM_BLOCKS, DAMPING, TELEPORT = 2, 0.85, 0.15


def link_rows(src, dst, n: int):
    """loadLinksMatrix's rows from 0-based (source, target) pairs, duplicates included: (ids, rowptr, cols, values) with
    row `page` holding 1.0 / (its number of pairs) at each distinct target."""
    src, dst = np.asarray(src, np.int64), np.asarray(dst, np.int64)
    ids, size = np.unique(src, return_counts=True)
    pairs = np.unique(src * n + dst)
    rows, cols = pairs // n, pairs % n
    per = np.searchsorted(rows, ids, side="right") - np.searchsorted(rows, ids, side="left")
    return ids, np.concatenate([[0], np.cumsum(per)]), cols, np.repeat(1.0 / size.astype(np.float64), per)


def literal_rows(lines, linkNum: int):
    """PageRank.loadLinksMatrix as written, on text lines: {page - 1: dense vector}."""
    groups = {}
    for line in lines:
        parts = re.split(r"\s+", line)
        while parts and parts[-1] == "":
            parts.pop()
        groups.setdefault(int(parts[0]), []).append(int(parts[1]))
    out = {}
    for page, links in groups.items():
        vec = np.zeros(linkNum)
        for l in links:
            vec[l - 1] = 1.0 / len(links)
        out[page - 1] = vec
    return out


def split(v: np.ndarray):
    """The re-split of the loop: 2 pieces of ceil(n / 2), the last taking the rest."""
    n = v.shape[0]
    s = int(math.ceil(n / NUM_BLOCKS))
    return [v[:s].copy(), v[s:].copy()]


def dense(rows: dict, n: int, iterations: int):
    """The example on the reference model: the final ranks pieces."""
    from oracle import reference_model as rm
    links = rm.DenseVecMatrix(sorted(rows.items()), n, n).transpose(NUM_BLOCKS).scalar("multiply", DAMPING)
    pieces = split(np.ones(n))
    r = np.ones(n) * TELEPORT
    for _ in range(iterations):
        res = links.multiply_dist_vector(rm.DistributedVector(list(enumerate(pieces)), n, NUM_BLOCKS)).vectors
        acc = res[0][1]
        for _, v in res[1:]:
            acc = acc + v
        pieces = split(acc + r)
    return pieces


class InLinks:
    """The in-link rows of every target, edges sorted by (target, source), with the position-major layout of the rows
    of in-degree <= light and one sequential accumulate per segment for the heavier rows."""

    def __init__(self, ids, rowptr, cols, vals, n: int, light: int = 4096):
        self.n = n
        self.seg = int(math.ceil(n / NUM_BLOCKS))
        src = np.repeat(np.asarray(ids, np.int64), np.diff(rowptr))
        tgt = np.asarray(cols, np.int64)
        w = np.asarray(vals, np.float64) * DAMPING
        order = np.lexsort((src, tgt))
        self.src, self.tgt, self.w = src[order], tgt[order], w[order]
        self.deg = np.bincount(self.tgt, minlength=n)
        self.start = np.concatenate([[0], np.cumsum(self.deg)])
        segid = self.src // self.seg
        self.new_seg = np.ones(len(self.src), bool)
        self.new_seg[1:] = (segid[1:] != segid[:-1]) | (self.tgt[1:] != self.tgt[:-1])
        few = np.flatnonzero(self.deg <= light)
        self.heavy = np.flatnonzero(self.deg > light)
        self.perm = few[np.argsort(-self.deg[few], kind="stable")]
        d = self.deg[self.perm]
        maxd = int(d.max()) if len(d) else 0
        self.counts = [int(np.searchsorted(-d, -k, side="right")) for k in range(1, maxd + 1)]     # rows with deg >= k
        self.edges = np.concatenate([self.start[self.perm[:c]] + k for k, c in enumerate(self.counts)]) if maxd \
            else np.zeros(0, np.int64)

    def step(self, x: np.ndarray, addend: float = TELEPORT) -> np.ndarray:
        p = self.w * x[self.src]
        y = np.empty(self.n)
        m = len(self.perm)
        tot, acc = np.zeros(m), np.zeros(m)
        off = 0
        for c in self.counts:
            e = self.edges[off:off + c]
            f = self.new_seg[e]
            if f.any():
                tot[:c][f] += acc[:c][f]
                acc[:c][f] = 0.0
            acc[:c] += p[e]
            off += c
        y[self.perm] = (tot + acc) + addend
        for i in self.heavy:
            a, b = self.start[i], self.start[i + 1]
            t = 0.0
            cuts = np.flatnonzero(self.new_seg[a:b]).tolist() + [b - a]
            for s0, s1 in zip(cuts[:-1], cuts[1:]):
                t = t + np.add.accumulate(np.concatenate([[0.0], p[a + s0:a + s1]]))[-1]
            y[i] = t + addend
        return y

    def run(self, iterations: int):
        x = np.ones(self.n)
        for _ in range(iterations):
            x = self.step(x)
        return split(x)


def rmat(scale: int, edge_factor: int, seed: int, abcd=(0.57, 0.19, 0.19, 0.05)):
    """Seeded R-MAT pairs (0-based source, target) over 2^scale pages."""
    rng = np.random.default_rng(seed)
    m = edge_factor << scale
    src = np.zeros(m, np.int64)
    dst = np.zeros(m, np.int64)
    a, b, c, _ = abcd
    for bit in range(scale):
        r = rng.random(m)
        src |= ((r >= a + b)).astype(np.int64) << bit
        dst |= (((r >= a) & (r < a + b)) | (r >= a + b + c)).astype(np.int64) << bit
    return src, dst


def random_graph(n: int, seed: int, mean_out: float = 4.0):
    """Uniform random pairs with duplicates, self-links, pages without out-links and pages without in-links."""
    rng = np.random.default_rng(seed)
    m = int(n * mean_out)
    src = rng.integers(0, n, m)
    dst = rng.integers(0, n, m)
    quiet = rng.random(n) < 0.2                          # about a fifth of the pages link nowhere
    keep = ~quiet[src]
    src, dst = src[keep], dst[keep]
    unreached = rng.random(n) < 0.2
    dst = np.where(unreached[dst], (dst + 1) % n, dst)
    dup = rng.integers(0, len(src), max(1, len(src) // 10))
    src = np.concatenate([src, src[dup], np.arange(0, n, 7)])
    dst = np.concatenate([dst, dst[dup], np.arange(0, n, 7)])             # duplicated lines and self-links
    return src, dst

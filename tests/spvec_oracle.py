"""Host restatement of SparseVecMatrix (matrix/SparseVecMatrix.scala) and randomSpaVecMatrix, the yardstick of the spvec
kernels.

A row set is a list of (id, indices, values).  `multiply_sparse` is multiplySparse in the library's fixed order: for each
row i of A, each stored k in order, each stored j of B(k, :): p = f32(A(i,k)) * f32(B(k,j)) in float32, C(i,j) = the
first p, then C(i,j) + p in float32.  numpy float32 scalars multiply and add with one IEEE rounding each and keep
subnormals, so a device result in the same order matches bit for bit.  `multiply_sparse_literal` is the reference's
dataflow (emit per k, join on k, reduceByKey) with the shuffle order as a parameter.
"""
from __future__ import annotations

from collections import defaultdict
from typing import Dict, List, Sequence, Tuple

import numpy as np

Rows = List[Tuple[int, np.ndarray, np.ndarray]]

# DistributedMatrixSuite.scala:27-32 and the expected product of "Sparse matrix multiply" (:152-162)
SUITE_ROWS = [(0, [1, 3], [2.0, 3.0]), (1, [0, 1], [5.0, 1.0]), (2, [3], [2.0]), (3, [1, 2], [1.0, 1.0])]
SUITE_PRODUCT = np.array([[10.0, 5.0, 3.0, 0.0], [5.0, 11.0, 0.0, 15.0], [0.0, 2.0, 2.0, 0.0], [5.0, 1.0, 0.0, 2.0]])


def multiply_sparse(A: Rows, B: Rows) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(rows, cols, float32 values) sorted by (row, col), in the fixed order described above."""
    brows = {int(i): (np.asarray(ix), np.asarray(v, np.float64)) for i, ix, v in B}
    out_r, out_c, out_v = [], [], []
    for i, aix, av in A:
        acc: Dict[int, np.float32] = {}
        for k, a in zip(np.asarray(aix), np.asarray(av, np.float64)):
            if int(k) not in brows:
                continue
            a32 = np.float32(a)
            bix, bv = brows[int(k)]
            for j, b in zip(bix, bv):
                p = np.float32(a32 * np.float32(b))
                acc[int(j)] = p if int(j) not in acc else np.float32(acc[int(j)] + p)
        for j in sorted(acc):
            out_r.append(int(i)); out_c.append(j); out_v.append(acc[j])
    order = np.lexsort((np.array(out_c, np.int64), np.array(out_r, np.int64))) if out_r else np.zeros(0, np.int64)
    return (np.array(out_r, np.int64)[order], np.array(out_c, np.int64)[order],
            np.array(out_v, np.float32).reshape(-1)[order])


def multiply_sparse_literal(A: Rows, B: Rows, rng: np.random.Generator = None) -> Dict[Tuple[int, int], np.float32]:
    """:22-50 as written: A's (k, (i, a.toFloat)) grouped by k, joined with B's (k, (j, b.toFloat)), products a * b in
    float32, reduceByKey(_ + _) in float32 over the products of a key in shuffle order (`rng` permutes it; None keeps
    the emit order).  Unmatched k are dropped; a key with one product keeps it as it is."""
    this = defaultdict(list)
    for i, aix, av in A:
        for k, a in zip(aix, av):
            this[int(k)].append((int(i), np.float32(a)))
    products = defaultdict(list)
    for k_, bix, bv in B:
        for j, b in zip(bix, bv):                      # otherEmits: (index, (j, b)) keyed by B's row id
            for i, a in this.get(int(k_), []):
                products[(i, int(j))].append(np.float32(a * np.float32(b)))
    out = {}
    for key, ps in products.items():
        if rng is not None:
            ps = [ps[t] for t in rng.permutation(len(ps))]
        acc = ps[0]
        for p in ps[1:]:
            acc = np.float32(acc + p)
        out[key] = acc
    return out


def to_dense(rows: Rows, n_rows: int, n_cols: int) -> np.ndarray:
    out = np.zeros((n_rows, n_cols))
    for i, ix, v in rows:
        out[i, np.asarray(ix, np.int64)] = v
    return out


def dense_to_rows(ids: Sequence[int], dense: np.ndarray) -> Rows:
    """DenseVecMatrix.toSparseVecMatrix (DenseVecMatrix.scala:1333-1353): the entries != 0 of each row in column order."""
    return [(int(i), np.flatnonzero(r != 0.0), r[r != 0.0]) for i, r in zip(ids, dense)]


# ---- randomSpaVecMatrix (the library's seeded column set; values as the reference) ----
def column_set(state0: int, first: int, n_cols: int, s: int) -> np.ndarray:
    """Selection sampling (Algorithm S) of s of n_cols columns from stream positions [first, first + n_cols) of the
    XORShift stream state0, taking column t when x * (n_cols - t) < q * 2^53; the sampler of mb_fill_sparse_uniform."""
    from oracle.reference_model import _xs_step
    st = state0 & ((1 << 64) - 1)
    for _ in range(2 * first):
        st = _xs_step(st)
    out, q = [], s
    for t in range(n_cols):
        if not q:
            break
        st = _xs_step(st)
        hi26 = st & ((1 << 26) - 1)
        st = _xs_step(st)
        x = (hi26 << 27) + (st & ((1 << 27) - 1))
        if x * (n_cols - t) < q << 53:
            out.append(t)
            q -= 1
    return np.array(out, np.int64)


def partition_rows(partition_seed: int, start: int, count: int, n_cols: int, s: int, lo: float = 0.0,
                   hi: float = 1.0) -> Rows:
    """The rows [start, start + count) of one partition: values at stream positions [0, s*count) (row r takes
    [r*s, (r+1)*s)), one column set drawn from positions [s*count, s*count + n_cols)."""
    from oracle import reference_model as rm
    cols = column_set(rm.hash_seed(partition_seed), s * count, n_cols, s)
    vals = rm.uniform_stream(partition_seed, 0, s * count, lo, hi).reshape(count, s)
    return [(start + r, cols, vals[r]) for r in range(count)]


def random_spa_vec_matrix(n_rows: int, n_cols: int, density: float, partitions: int, seed: int) -> Rows:
    from oracle import reference_model as rm
    s = int(float(n_cols) * float(density))
    seeds = rm.java_random_longs(seed, partitions)
    out, start = [], 0
    for p in range(partitions):
        end = ((p + 1) * n_rows) // partitions
        out += partition_rows(seeds[p], start, end - start, n_cols, s)
        start = end
    return out

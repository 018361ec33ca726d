"""Host restatement of the reference's sparse-block code, the yardstick of the sparse kernels.

Each function restates one loop of matrix/Matrices.scala or matrix/LibMatrixMult.scala in the same order, with numpy
doing element-wise IEEE multiplies and adds (never fused), so a device result that follows the same order must match it
bit for bit.  A CSC block is a tuple (rows, cols, colptr, rowidx, values).  multSparseDense is restated twice: as written
(with the `bi` that should be `bk` at LibMatrixMult.scala:60) and corrected.
"""
from __future__ import annotations

from typing import Tuple

import numpy as np

Csc = Tuple[int, int, np.ndarray, np.ndarray, np.ndarray]


def csc_from_dense_pattern(dense: np.ndarray, mask: np.ndarray) -> Csc:
    """The CSC block storing dense[r, c] wherever mask[r, c] (explicit zeros included), rows ascending."""
    rows, cols = dense.shape
    colptr = np.zeros(cols + 1, dtype=np.int32)
    ri, va = [], []
    for j in range(cols):
        r = np.nonzero(mask[:, j])[0]
        ri.append(r.astype(np.int32))
        va.append(dense[r, j].astype(np.float64))
        colptr[j + 1] = colptr[j] + r.size
    cat = lambda xs, dt: np.concatenate(xs).astype(dt) if xs else np.zeros(0, dt)
    return rows, cols, colptr, cat(ri, np.int32), cat(va, np.float64)


def random_csc(rng: np.random.Generator, rows: int, cols: int, density: float, empty_cols: float = 0.0) -> Csc:
    mask = rng.random((rows, cols)) < density
    if empty_cols:
        mask[:, rng.random(cols) < empty_cols] = False
    return csc_from_dense_pattern(rng.standard_normal((rows, cols)), mask)


def to_dense(S: Csc) -> np.ndarray:
    """SparseMatrix.toDense (Matrices.scala:106-119)."""
    rows, cols, cp, ri, va = S
    c = np.zeros((rows, cols), order="F")
    for j in range(cols):
        c[ri[cp[j]:cp[j + 1]], j] = va[cp[j]:cp[j + 1]]
    return c


def mult_dense_sparse(A: np.ndarray, B: Csc) -> np.ndarray:
    """LibMatrixMult.multDenseSparse (:15-41), including the copy of a column holding exactly one 1.0 (:28-29)."""
    _, n, cp, ri, va = B
    m = A.shape[0]
    c = np.zeros((m, n), order="F")
    for j in range(n):
        p0, p1 = cp[j], cp[j + 1]
        if p1 - p0 == 1 and va[p0] == 1.0:
            c[:, j] = A[:, ri[p0]]
            continue
        for p in range(p0, p1):
            c[:, j] = c[:, j] + va[p] * A[:, ri[p]]
    return c


def _column_vectors(A: Csc):
    _, cols, cp, ri, va = A
    return [(ri[cp[k]:cp[k + 1]], va[cp[k]:cp[k + 1]]) for k in range(cols)]


def mult_sparse_dense_literal(A: Csc, B: np.ndarray) -> np.ndarray:
    """LibMatrixMult.multSparseDense (:43-77) as written.  `b` is B's column-major data array; an index past its end
    raises IndexError where the JVM throws ArrayIndexOutOfBoundsException."""
    m, cd = A[0], A[1]
    n = B.shape[1]
    b = np.asfortranarray(B).reshape(-1, order="F")
    a = _column_vectors(A)
    c = np.zeros(m * n)
    for bi in range(0, n, 32):
        for bk in range(0, cd, 32):
            bimin = min(n, bi + 32)
            bklen = min(cd, bk + 32) - bk
            for i in range(bi, bimin):
                bixi = i * cd + bi
                cixj = i * m
                for k in range(bklen):
                    if bixi + k >= b.size:
                        raise IndexError(bixi + k)
                    value = b[bixi + k]
                    aix, avals = a[bk + k]
                    c[cixj + aix] = c[cixj + aix] + value * avals
    return c.reshape((m, n), order="F")


def mult_sparse_dense(A: Csc, B: np.ndarray) -> np.ndarray:
    """The same loop with `bk` at :60: C(r, i) summed over k ascending."""
    m, cd = A[0], A[1]
    c = np.zeros((m, B.shape[1]), order="F")
    for k, (aix, avals) in enumerate(_column_vectors(A)):
        if aix.size:
            c[aix, :] = c[aix, :] + B[k, :][None, :] * avals[:, None]
    return c


def spgemm(A: Csc, B: Csc) -> np.ndarray:
    """SparseMatrix.multiply (Matrices.scala:129-152): for each stored k of B(:, j) in order, c(aix) += bval * a."""
    m = A[0]
    _, n, cp, ri, va = B
    acols = _column_vectors(A)
    c = np.zeros((m, n), order="F")
    for j in range(n):
        for p in range(cp[j], cp[j + 1]):
            aix, avals = acols[ri[p]]
            if aix.size:
                c[aix, j] = c[aix, j] + va[p] * avals
    return c


# ---- the sparse generator (mb_fill_sparse_uniform), stepped sequentially: independent of the device's jump tables ----
def sample_rows(state0: int, rows: int, cols: int, s: int) -> np.ndarray:
    """Row indices (cols x s) of a block whose stream starts at state0: column j runs Algorithm S over positions
    [s*cols + j*rows, +rows), taking row t when x * (rows - t) < q * 2^53."""
    from oracle.reference_model import _xs_step
    st = state0 & ((1 << 64) - 1)
    for _ in range(2 * s * cols):
        st = _xs_step(st)
    out = np.zeros((cols, s), dtype=np.int32)
    for j in range(cols):
        q = s
        for t in range(rows):
            st = _xs_step(st)
            hi26 = st & ((1 << 26) - 1)
            st = _xs_step(st)
            x = (hi26 << 27) + (st & ((1 << 27) - 1))
            if q and x * (rows - t) < q << 53:
                out[j, s - q] = t
                q -= 1
    return out


def sparse_block(partition_seed: int, rows: int, cols: int, s: int) -> Csc:
    from oracle import reference_model as rm
    ri = sample_rows(rm.hash_seed(partition_seed), rows, cols, s)
    vals = rm.uniform_stream(partition_seed, 0, s * cols)
    colptr = (np.arange(cols + 1) * s).astype(np.int32)
    return rows, cols, colptr, ri.reshape(-1), vals


def column_count(cols: int, density: float) -> int:
    """`(numCols * sparsity).toInt` (Matrices.scala:161)."""
    return int(float(cols) * float(density))

"""CPU restatement of DenseVecMatrix.computeSVD (matrix/DenseVecMatrix.scala:1444-1652, 1685-1834), step by step:
dspr into a packed upper triangle per row, `+=` over partitions, triuToFull; the mode chooser and its requires; LAPACK's
dgesdd (scipy, lapack_driver="gesdd") for local-svd and ARPACK's dsaupd/dseupd (scipy.sparse.linalg.eigsh, which="LM",
ncv = min(2k, n)) for the eigs modes; the effective rank; N = V_k S_k^-1 and U = A N.  The test suite's yardstick for the
device path; nothing under marlin_b200/ imports it."""
from __future__ import annotations

from typing import List, Optional, Tuple

import numpy as np
import scipy.linalg
import scipy.sparse.linalg


def _partitions(rows, parts: int):
    """sc.parallelize(rows, parts): contiguous slices."""
    n = len(rows)
    return [rows[(i * n) // parts:((i + 1) * n) // parts] for i in range(parts)]


def compute_gramian_matrix(rows, n: int, partitions: int = 2) -> np.ndarray:
    """:1464-1486 — per partition dspr("U", n, 1.0, v, U) for every row, partitions combined with `+=`, then triuToFull."""
    if n > 65535:
        raise ValueError(f"Argument with more than 65535 cols: {n}")
    nt = (n // 2) * (n + 1) if n % 2 == 0 else n * ((n + 1) // 2)
    cols = np.concatenate([np.full(c + 1, c) for c in range(n)]) if n else np.zeros(0, dtype=int)
    rws = np.concatenate([np.arange(c + 1) for c in range(n)]) if n else np.zeros(0, dtype=int)
    total = None
    for part in _partitions(list(rows), partitions):
        U = np.zeros(nt)
        for _, v in part:
            v = np.asarray(v, dtype=np.float64)
            U += v[rws] * v[cols]                       # dspr: U(i, j) += alpha * x(i) * x(j), i <= j, column-major packed
        total = U if total is None else total + U
    G = np.zeros((n, n))
    G[rws, cols] = total
    G[cols, rws] = total
    return G


def multiply_gramian_matrix_by(rows, v: np.ndarray, partitions: int = 2) -> np.ndarray:
    """:1444-1459 — sum over rows of (r . v) r per partition (as A_p^T (A_p v)), partitions combined with `+=`."""
    total = None
    for part in _partitions(list(rows), partitions):
        U = np.zeros(v.shape[0])
        if part:
            Ap = np.array([r for _, r in part])
            U += Ap.T @ (Ap @ v)
        total = U if total is None else total + U
    return total


def svd_mode(n: int, k: int, mode: str) -> str:
    """:1565-1604 plus the column cap of computeGramianMatrix; messages as in the reference."""
    if not (0 < k <= n):
        raise ValueError(f"Request up to n singular values but got k={k} and n={n}.")
    if mode == "auto":
        if n < 100 or k > n // 2:
            cm = "local-eigs" if k < n // 3 else "local-svd"
        else:
            cm = "dist-eigs"
    elif mode in ("local-svd", "local-eigs", "dist-eigs"):
        cm = mode
    else:
        raise ValueError(f"Do not support mode {mode}.")
    if cm != "local-svd" and not k < n:
        raise ValueError(f"k must be smaller than n in {cm} mode but got k={k} and n={n}.")
    if n > 65535:
        raise ValueError(f"Argument with more than 65535 cols: {n}")
    return cm


def effective_rank(sigmas: np.ndarray, k: int, r_cond: float) -> int:
    """:1607-1621"""
    if len(sigmas) == 0:
        return 0
    threshold = r_cond * sigmas[0]
    i = 0
    while i < min(k, len(sigmas)) and sigmas[i] >= threshold:
        i += 1
    return i


def symmetric_eigs(mul, n: int, k: int, tol: float, max_iter: int) -> Tuple[np.ndarray, np.ndarray]:
    """EigenValueDecomposition.symmetricEigs (:1725-1834): ARPACK, which="LM", ncv = min(2k, n), pairs sorted by
    eigenvalue descending."""
    if not n > k:
        raise ValueError(f"Number of required eigenvalues {k} must be smaller than matrix dimension {n}")
    op = scipy.sparse.linalg.LinearOperator((n, n), matvec=lambda x: mul(np.asarray(x).reshape(-1)), dtype=np.float64)
    d, z = scipy.sparse.linalg.eigsh(op, k=k, which="LM", ncv=min(2 * k, n), tol=tol, maxiter=max_iter)
    order = np.argsort(-d, kind="stable")
    return d[order], z[:, order]


def compute_svd(rows, n: int, k: int, compute_u: bool = False, r_cond: float = 1e-9, max_iter: Optional[int] = None,
                tol: float = 1e-10, mode: str = "auto", partitions: int = 2):
    """:1531-1652 -> (U as a list of (index, row) or None, s, V (n x sk))."""
    rows = [(int(i), np.asarray(v, dtype=np.float64)) for i, v in rows]
    if max_iter is None:
        max_iter = max(300, k * 3)
    cm = svd_mode(n, k, mode)
    if cm == "local-eigs":
        G = compute_gramian_matrix(rows, n, partitions)
        sigma_sq, u = symmetric_eigs(lambda v: G @ v, n, k, tol, max_iter)
    elif cm == "local-svd":
        G = compute_gramian_matrix(rows, n, partitions)
        u, sigma_sq, _ = scipy.linalg.svd(G, lapack_driver="gesdd")
    else:
        sigma_sq, u = symmetric_eigs(lambda v: multiply_gramian_matrix_by(rows, v, partitions), n, k, tol, max_iter)
    sigmas = np.sqrt(sigma_sq)
    sk = effective_rank(sigmas, k, r_cond)
    s = sigmas[:sk].copy()
    V = np.asfortranarray(u[:, :sk])
    if not compute_u:
        return None, s, V
    N = V.copy()
    for j in range(sk):
        N[:, j] /= sigmas[j]
    return [(i, r @ N) for i, r in rows], s, V

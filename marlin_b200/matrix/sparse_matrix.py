"""Sparse blocks: the reference's local SparseVector / SparseMatrix (matrix/Vectors.scala:217-229,
matrix/Matrices.scala:57-173) and their device form, a CSC block behind the C ABI.

A SparseMatrix is one SparseVector per column.  On the device it is CSC: `colptr` int32[cols+1], `rowidx` int32[nnz],
`values` f64[nnz], held in torch tensors (so NCCL can move them) and checked on the way in: row indices must lie in
[0, rows) and increase strictly within each column, where the reference accepts unsorted or repeated indices unchecked.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from .. import _native as nat
from ..runtime import Runtime


class SparseVector:
    """Vectors.scala:217-229: `size`, sorted `indices` and their `values`."""

    def __init__(self, size: int, indices: Sequence[int], values: Sequence[float]):
        self.length = int(size)
        self.indices = np.asarray(indices, dtype=np.int32).reshape(-1)
        self.values = np.asarray(values, dtype=np.float64).reshape(-1)
        if self.indices.shape != self.values.shape:
            raise ValueError("SparseVector: indices and values differ in length")

    @property
    def size(self) -> int:
        return self.length

    def isEmpty(self) -> bool:
        return self.length == 0


class SparseMatrix:
    """Matrices.scala:57-173: numRows x numCols, `values` = one SparseVector per column.  `toDense` and `multiply` run on
    the GPU through a sparse block."""

    def __init__(self, numRows: int, numCols: int, values: Sequence[Optional[SparseVector]]):
        self.numRows, self.numCols = int(numRows), int(numCols)
        self.values: List[Optional[SparseVector]] = list(values)
        if len(self.values) != self.numCols:
            raise ValueError(f"SparseMatrix: {len(self.values)} column vectors for {self.numCols} columns")

    def to_csc(self) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """(colptr, rowidx, values) host arrays, checked (mb_sparse_check)."""
        cols = [v if v is not None else SparseVector(self.numRows, [], []) for v in self.values]
        counts = np.array([len(v.indices) for v in cols], dtype=np.int64)
        if counts.sum() > 2**31 - 1:
            raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, f"sparse block with {counts.sum()} non-zeros: at most 2^31 - 1")
        colptr = np.zeros(self.numCols + 1, dtype=np.int32)
        colptr[1:] = np.cumsum(counts)
        rowidx = np.concatenate([v.indices for v in cols]).astype(np.int32) if cols else np.zeros(0, np.int32)
        vals = np.concatenate([v.values for v in cols]).astype(np.float64) if cols else np.zeros(0)
        check_csc(self.numRows, self.numCols, colptr, rowidx)
        return colptr, rowidx, vals

    def toDense(self) -> np.ndarray:
        """Matrices.scala:106-119"""
        from .sub_matrix import SubMatrix
        return SubMatrix(spMatrix=self).toBreeze()

    def multiply(self, other: "SparseMatrix") -> np.ndarray:
        """Matrices.scala:129-152: sparse x sparse, a dense result."""
        from .sub_matrix import SubMatrix
        return SubMatrix(spMatrix=self).multiply(SubMatrix(spMatrix=other)).toBreeze()


def check_csc(rows: int, cols: int, colptr: np.ndarray, rowidx: np.ndarray) -> None:
    """The structure checks of mb_sparse_upload (pure host logic of the library)."""
    cp = np.ascontiguousarray(colptr, dtype=np.int32)
    ri = np.ascontiguousarray(rowidx, dtype=np.int32)
    if cp.shape != (cols + 1,):
        raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, f"sparse block: colptr has {cp.size} entries, expected {cols + 1}")
    if int(cp[-1]) != ri.size:
        raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, f"sparse block: colptr ends at {int(cp[-1])}, nnz is {ri.size}")
    nat.check(nat.load().mb_sparse_check(rows, cols, cp.ctypes.data, ri.ctypes.data if ri.size else None))


def column_count(rows: int, cols: int, density: float) -> int:
    """Non-zeros per column of a sparse randomBlockMatrix block: `(numCols * sparsity).toInt` (Matrices.scala:161), with
    density <= 0 and s > rows rejected (mb_sparse_column_count)."""
    s = C.c_int32()
    nat.check(nat.load().mb_sparse_column_count(rows, cols, float(density), C.byref(s)))
    return int(s.value)


class SparseBlock:
    """Device CSC storage of one sparse SubMatrix.  Immutable: the scalar ops make a new values array and share the
    structure; the library caches a CSR copy with the handle for sparse x dense products."""

    def __init__(self, rows: int, cols: int, colptr: torch.Tensor, rowidx: torch.Tensor, values: torch.Tensor):
        self.rows, self.cols = int(rows), int(cols)
        self.colptr, self.rowidx, self.values = colptr, rowidx, values
        self.nnz = int(values.numel())
        self._handle = None

    @staticmethod
    def from_host(rows: int, cols: int, colptr: np.ndarray, rowidx: np.ndarray, values: np.ndarray, device=None) -> "SparseBlock":
        check_csc(rows, cols, colptr, rowidx)
        if device is None:
            device = Runtime.get().device if Runtime.available() else torch.device("cpu")
        t = lambda a, dt: torch.tensor(np.ascontiguousarray(a, dtype=dt), device=device)
        return SparseBlock(rows, cols, t(colptr, np.int32), t(rowidx, np.int32), t(values, np.float64))

    @staticmethod
    def empty(rows: int, cols: int, nnz: int, device=None) -> "SparseBlock":
        if device is None:
            device = Runtime.get().device
        return SparseBlock(rows, cols, torch.empty(cols + 1, dtype=torch.int32, device=device),
                           torch.empty(nnz, dtype=torch.int32, device=device), torch.empty(nnz, dtype=torch.float64, device=device))

    def with_values(self, values: torch.Tensor) -> "SparseBlock":
        return SparseBlock(self.rows, self.cols, self.colptr, self.rowidx, values)

    def handle(self):
        if self._handle is None:
            if not self.values.is_cuda:
                raise nat.MarlinError(nat.MB_ERR_CUDA, "sparse block lives in host memory: marlin_b200 computes on H100 only "
                                      "(no CPU fallback)")
            rt = Runtime.get()
            h = nat.c_sp()
            ptr = lambda t: C.c_void_p(t.data_ptr()) if t.numel() else None
            nat.check(rt.lib.mb_sparse_wrap(rt.ctx, self.rows, self.cols, self.nnz, ptr(self.colptr), ptr(self.rowidx),
                                            ptr(self.values), C.byref(h)))
            self._handle = h
        return self._handle

    def to_host(self) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        return self.colptr.cpu().numpy(), self.rowidx.cpu().numpy(), self.values.cpu().numpy()

    def toSparseMatrix(self) -> SparseMatrix:
        cp, ri, va = self.to_host()
        return SparseMatrix(self.rows, self.cols, [SparseVector(self.rows, ri[cp[j]:cp[j + 1]], va[cp[j]:cp[j + 1]])
                                                   for j in range(self.cols)])

    # ---- one packed buffer per tile for comm.exchange: values, then colptr, then rowidx (8-byte aligned values) ----
    def pack(self) -> torch.Tensor:
        as_bytes = lambda t: t.view(torch.uint8) if t.numel() else torch.empty(0, dtype=torch.uint8, device=t.device)
        return torch.cat([as_bytes(self.values), as_bytes(self.colptr), as_bytes(self.rowidx)])

    @staticmethod
    def packed_bytes(cols: int, nnz: int) -> int:
        return 8 * nnz + 4 * (cols + 1) + 4 * nnz

    @staticmethod
    def unpack(buf: torch.Tensor, rows: int, cols: int, nnz: int) -> "SparseBlock":
        v = buf[: 8 * nnz].view(torch.float64)
        cp = buf[8 * nnz: 8 * nnz + 4 * (cols + 1)].view(torch.int32)
        ri = buf[8 * nnz + 4 * (cols + 1):].view(torch.int32)
        return SparseBlock(rows, cols, cp, ri, v)

    def __del__(self):
        h = getattr(self, "_handle", None)
        if h is not None:
            try:
                rt = Runtime._instance
                if rt is not None:
                    rt.lib.mb_sparse_free(rt.ctx, h)
            except Exception:
                pass

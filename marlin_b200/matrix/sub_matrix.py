"""SubMatrix — the per-block value type (matrix/SubMatrix.scala), device resident.

The reference's SubMatrix wraps a Breeze DenseMatrix[Double] on the JVM heap; here the same
(data, offset, rows, cols, majorStride, isTranspose) record points into HBM.  The buffer is a torch
tensor only so that torch.distributed (NCCL) can move it; every arithmetic method calls the C ABI
of libmarlin_b200.so (the kernel seam named in SURVEY.md §2 #3).  A sparse block (`SubMatrix(spMatrix=...)`) holds a
device CSC block instead (sparse_matrix.SparseBlock); multiply dispatches the four sparsity pairs as the reference does
(:87-119) and the scalar ops change only the stored values (:52-58, 71-85, 121-129).
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Union

import numpy as np
import torch

from .. import _native as nat
from ..runtime import Runtime
from .sparse_matrix import SparseBlock, SparseMatrix

_TORCH_DTYPE = {nat.MB_F64: torch.float64, nat.MB_BF16: torch.bfloat16, nat.MB_F32: torch.float32}
_MB_DTYPE = {v: k for k, v in _TORCH_DTYPE.items()}

Number = Union[int, float]


class SubMatrix:
    """A dense block.  Element (r, c) = buf.flatten()[offset + r + c*ld] (or [offset + c + r*ld] if
    is_transpose), exactly Breeze's DenseMatrix indexing."""

    def __init__(self, denseMatrix=None, *, spMatrix: Optional[SparseMatrix] = None, sparse: Optional[SparseBlock] = None,
                 buf: Optional[torch.Tensor] = None, rows: int = 0, cols: int = 0,
                 ld: Optional[int] = None, offset: int = 0, is_transpose: bool = False, device=None):
        self._handle = None
        self._sparse: Optional[SparseBlock] = None
        if spMatrix is not None:
            sparse = SparseBlock.from_host(spMatrix.numRows, spMatrix.numCols, *spMatrix.to_csc(), device=device)
        if sparse is not None:
            self._sparse = sparse
            self.buf = None
            self._rows, self._cols = sparse.rows, sparse.cols
            self.ld, self.offset, self.is_transpose = max(1, sparse.rows), 0, False
            return
        if denseMatrix is not None:
            if isinstance(denseMatrix, SubMatrix):
                src = denseMatrix
                buf, rows, cols, ld, offset, is_transpose = src.buf, src._rows, src._cols, src.ld, src.offset, src.is_transpose
            else:
                arr = np.asarray(denseMatrix, dtype=np.float64)
                if arr.ndim != 2:
                    raise ValueError("SubMatrix needs a 2-D dense matrix")
                rows, cols = arr.shape
                flat = np.ascontiguousarray(arr.T).reshape(-1)            # column-major data array
                t = torch.from_numpy(flat)
                if device is None:
                    device = Runtime.get().device if Runtime.available() else torch.device("cpu")
                buf = t.to(device)
                ld, offset, is_transpose = max(1, rows), 0, False
        if buf is None:
            raise ValueError("SubMatrix: no data")
        if not buf.is_contiguous():
            raise ValueError("SubMatrix buffer must be contiguous")
        self.buf = buf
        self._rows, self._cols = int(rows), int(cols)
        self.ld = int(ld if ld is not None else max(1, (cols if is_transpose else rows)))
        self.offset = int(offset)
        self.is_transpose = bool(is_transpose)

    # ---- construction helpers ----
    @staticmethod
    def empty(rows: int, cols: int, dtype: int = nat.MB_F64, device=None) -> "SubMatrix":
        if device is None:
            device = Runtime.get().device
        buf = torch.empty(max(1, rows) * max(0, cols) if rows * cols else 0, dtype=_TORCH_DTYPE[dtype], device=device)
        return SubMatrix(buf=buf, rows=rows, cols=cols, ld=max(1, rows))

    @staticmethod
    def zeros(rows: int, cols: int, dtype: int = nat.MB_F64, device=None) -> "SubMatrix":
        out = SubMatrix.empty(rows, cols, dtype, device)
        out.buf.zero_()
        return out

    # ---- reference accessors (matrix/SubMatrix.scala:27-39) ----
    @property
    def rows(self) -> int:
        return self._rows

    @property
    def cols(self) -> int:
        return self._cols

    @property
    def isSparse(self) -> bool:
        return self._sparse is not None

    @property
    def sparseBlock(self) -> SparseBlock:
        if self._sparse is None:
            raise nat.MarlinArgumentError(nat.MB_ERR_UNSUPPORTED, "sparseBlock of a dense block")
        return self._sparse

    @property
    def denseBlock(self) -> "SubMatrix":
        self._dense_only("denseBlock")
        return self

    def _dense_only(self, what: str) -> None:
        if self._sparse is not None:
            raise nat.MarlinArgumentError(nat.MB_ERR_UNSUPPORTED, f"{what} is not supported on sparse blocks: call "
                                          "toDenseBlocks first")

    def toDense(self) -> "SubMatrix":
        """SparseMatrix.toDense (Matrices.scala:106-119) as a packed column-major block; a dense block is returned as is."""
        if self._sparse is None:
            return self
        rt = Runtime.get(); rt.sync_stream()
        out = SubMatrix.empty(self._rows, self._cols, nat.MB_F64, self._sparse.values.device)
        nat.check(rt.lib.mb_sparse_to_dense(rt.ctx, self._sparse.handle(), out.handle()))
        return out

    @property
    def dtype(self) -> int:
        return nat.MB_F64 if self._sparse is not None else _MB_DTYPE[self.buf.dtype]

    @property
    def t(self) -> "SubMatrix":
        """Breeze `.t`: a transposed view, no copy."""
        self._dense_only("transpose")
        return SubMatrix(buf=self.buf, rows=self._cols, cols=self._rows, ld=self.ld, offset=self.offset,
                         is_transpose=not self.is_transpose)

    def slice(self, r0: int, r1: int, c0: int, c1: int) -> "SubMatrix":
        """Breeze `m(r0 until r1, c0 until c1)`: a view with the parent's majorStride (BlockMatrix.scala:198,299)."""
        self._dense_only("slice")
        if not (0 <= r0 <= r1 <= self._rows and 0 <= c0 <= c1 <= self._cols):
            raise ValueError("slice out of range")
        rs, cs = (self.ld, 1) if self.is_transpose else (1, self.ld)
        return SubMatrix(buf=self.buf, rows=r1 - r0, cols=c1 - c0, ld=self.ld, offset=self.offset + r0 * rs + c0 * cs,
                         is_transpose=self.is_transpose)

    def is_packed(self) -> bool:
        return self._sparse is None and (not self.is_transpose) and self.offset == 0 and self.ld == max(1, self._rows)

    # ---- native handle ----
    def handle(self):
        """The dense block handle; every dense-only operation goes through here."""
        self._dense_only("this operation")
        if self._handle is None:
            if not self.buf.is_cuda:
                raise nat.MarlinError(nat.MB_ERR_CUDA, "block lives in host memory: marlin_b200 computes on H100 only "
                                      "(no CPU fallback)")
            rt = Runtime.get()
            h = nat.c_blk()
            nat.check(rt.lib.mb_block_wrap(rt.ctx, C.c_void_p(self.buf.data_ptr()), self.offset, self._rows, self._cols,
                                           self.ld, int(self.is_transpose), self.dtype, C.byref(h)))
            self._handle = h
            ev = getattr(self, "_ready_event", None)
            if ev is not None:
                nat.check(rt.lib.mb_block_set_ready_event(h, C.c_void_p(ev.cuda_event)))
        return self._handle

    def mark_ready(self) -> "SubMatrix":
        """Record that everything queued so far on the current stream produces this block's FINAL contents (blocks are
        immutable values, like the blocks of a cached RDD): the multi-GPU multiply then offers the block to other ranks as
        soon as this event completes instead of after all later work on the stream (see mb_block_set_ready_event)."""
        if self.buf is not None and self.buf.is_cuda:
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(self.buf.device))
            self._ready_event = ev
            if self._handle is not None:
                rt = Runtime.get()
                nat.check(rt.lib.mb_block_set_ready_event(self._handle, C.c_void_p(ev.cuda_event)))
        return self

    def __del__(self):
        h = getattr(self, "_handle", None)
        if h is not None:
            try:
                rt = Runtime._instance
                if rt is not None:
                    rt.lib.mb_block_free(rt.ctx, h)
            except Exception:
                pass

    def _new_like(self, rows: Optional[int] = None, cols: Optional[int] = None, dtype: Optional[int] = None) -> "SubMatrix":
        """Result block for an element-wise op: same shape and the same storage orientation as `self`
        (a row-major DenseVecMatrix shard stays row-major, so the kernels take the flat 128-bit path)."""
        rows = self._rows if rows is None else rows
        cols = self._cols if cols is None else cols
        dtype = self.dtype if dtype is None else dtype
        if self.is_transpose:
            buf = torch.empty(rows * cols, dtype=_TORCH_DTYPE[dtype], device=self.buf.device)
            return SubMatrix(buf=buf, rows=rows, cols=cols, ld=max(1, cols), is_transpose=True)
        return SubMatrix.empty(rows, cols, dtype, self.buf.device)

    # ---- arithmetic (matrix/SubMatrix.scala:41-139) ----
    def _values_block(self) -> "SubMatrix":
        """The stored values of a sparse block as an nnz x 1 dense block."""
        v = self._sparse.values
        return SubMatrix(buf=v, rows=v.numel(), cols=1, ld=max(1, v.numel()))

    def _sparse_values_op(self, op) -> "SubMatrix":
        """A scalar op on a sparse block: the reference maps only the stored values (:52-58, 71-85, 121-129), so the
        result keeps the pattern (a sparse block plus 1 is not A + 1).  Runs the dense element-wise kernel on them."""
        vals = self._values_block()
        res = op(vals) if vals.rows else vals
        return SubMatrix(sparse=self._sparse.with_values(res.buf if vals.rows else self._sparse.values.clone()))

    def _check_both_dense(self, other: "SubMatrix", opname: str) -> None:
        if self.isSparse or other.isSparse:
            raise nat.MarlinArgumentError(nat.MB_ERR_UNSUPPORTED, f"Not supported {opname}-operator between matrices of "
                                          f"sparsity with {str(self.isSparse).lower()} and {str(other.isSparse).lower()}")

    def add(self, other: Union["SubMatrix", Number]) -> "SubMatrix":
        if isinstance(other, SubMatrix):
            self._check_both_dense(other, "add")
        elif self.isSparse:
            return self._sparse_values_op(lambda v: v.add(other))
        rt = Runtime.get(); rt.sync_stream()
        out = self._new_like()
        if isinstance(other, SubMatrix):
            nat.check(rt.lib.mb_block_add(rt.ctx, self.handle(), other.handle(), out.handle()))      # :41-45
        else:
            nat.check(rt.lib.mb_block_axpb(rt.ctx, self.handle(), 1.0, float(other), out.handle()))   # :52-58
        return out

    def subtract(self, other: Union["SubMatrix", Number]) -> "SubMatrix":
        if isinstance(other, SubMatrix):
            self._check_both_dense(other, "subtract")
        elif self.isSparse:
            return self._sparse_values_op(lambda v: v.subtract(other))
        rt = Runtime.get(); rt.sync_stream()
        out = self._new_like()
        if isinstance(other, SubMatrix):
            nat.check(rt.lib.mb_block_sub(rt.ctx, self.handle(), other.handle(), out.handle()))      # :60-64
        else:
            nat.check(rt.lib.mb_block_axpb(rt.ctx, self.handle(), 1.0, -float(other), out.handle()))  # :71-77
        return out

    def divide(self, b: Number) -> "SubMatrix":
        if self.isSparse:
            return self._sparse_values_op(lambda v: v.divide(b))
        rt = Runtime.get(); rt.sync_stream()
        out = self._new_like()
        nat.check(rt.lib.mb_block_div(rt.ctx, self.handle(), float(b), 0, out.handle()))               # :79-85
        return out

    def _divide_into(self, b: Number, out: "SubMatrix") -> None:
        """out := this / b (IEEE division) into an existing view."""
        rt = Runtime.get(); rt.sync_stream()
        nat.check(rt.lib.mb_block_div(rt.ctx, self.handle(), float(b), 0, out.handle()))

    def subtractBy(self, b: Number) -> "SubMatrix":
        """b - x (matrix/BlockMatrix.scala:414-424; returns a new block instead of mutating in place)."""
        rt = Runtime.get(); rt.sync_stream()
        out = self._new_like()
        nat.check(rt.lib.mb_block_axpb(rt.ctx, self.handle(), -1.0, float(b), out.handle()))
        return out

    def divideBy(self, b: Number) -> "SubMatrix":
        """b / x (matrix/BlockMatrix.scala:442-452)."""
        rt = Runtime.get(); rt.sync_stream()
        out = self._new_like()
        nat.check(rt.lib.mb_block_div(rt.ctx, self.handle(), float(b), 1, out.handle()))
        return out

    def elementMultiply(self, other: "SubMatrix") -> "SubMatrix":
        rt = Runtime.get(); rt.sync_stream()
        out = self._new_like()
        nat.check(rt.lib.mb_block_hadamard(rt.ctx, self.handle(), other.handle(), out.handle()))
        return out

    def multiply(self, other, out: Optional["SubMatrix"] = None, accumulate: bool = False,
                 out_dtype: Optional[int] = None) -> "SubMatrix":
        """:87-111 (block x block, block x local matrix) and :123-131 (scalar).  With a sparse side the product is dense:
        multDenseSparse, multSparseDense (the true product; the reference's loop is right only for K, N <= 32) or
        SparseMatrix.multiply, each summed in the reference's order (see include/marlin_b200.h)."""
        rt = Runtime.get(); rt.sync_stream()
        if isinstance(other, (int, float)):
            if self.isSparse:
                return self._sparse_values_op(lambda v: v.multiply(float(other)))
            res = self._new_like()
            nat.check(rt.lib.mb_block_axpb(rt.ctx, self.handle(), float(other), 0.0, res.handle()))
            return res
        if not isinstance(other, SubMatrix):
            other = SubMatrix(other, device=self.device)
        if self.isSparse or other.isSparse:
            if out is None:
                if accumulate:
                    raise ValueError("accumulate needs an output block")
                out = SubMatrix.empty(self._rows, other._cols, nat.MB_F64, self.device)
            if self.isSparse and other.isSparse:
                nat.check(rt.lib.mb_spgemm_dense_out(rt.ctx, self._sparse.handle(), other._sparse.handle(), out.handle(),
                                                     int(accumulate)))
            elif self.isSparse:
                nat.check(rt.lib.mb_spmm_sparse_dense(rt.ctx, self._sparse.handle(), other.handle(), out.handle(),
                                                      int(accumulate)))
            else:
                nat.check(rt.lib.mb_spmm_dense_sparse(rt.ctx, self.handle(), other._sparse.handle(), out.handle(),
                                                      int(accumulate)))
            return out
        if out is None:
            if accumulate:
                raise ValueError("accumulate needs an output block")
            dt = out_dtype if out_dtype is not None else (nat.MB_F32 if self.dtype == nat.MB_BF16 else self.dtype)
            out = SubMatrix.empty(self._rows, other._cols, dt, self.buf.device)
        nat.check(rt.lib.mb_block_gemm(rt.ctx, self.handle(), other.handle(), out.handle(), int(accumulate)))
        return out

    def dot(self, other: "SubMatrix") -> float:
        """Breeze `v.t * w` of two single-column (or single-row) blocks (matrix/DistributedVector.scala:167)."""
        rt = Runtime.get(); rt.sync_stream()
        out = C.c_double()
        nat.check(rt.lib.mb_block_dot(rt.ctx, self.handle(), other.handle(), C.byref(out)))
        return float(out.value)

    def outer(self, other: "SubMatrix") -> "SubMatrix":
        """Breeze `v * w.t` (matrix/DistributedVector.scala:157): rank-1 block of two vectors."""
        rt = Runtime.get(); rt.sync_stream()
        n0 = self._rows * self._cols
        n1 = other._rows * other._cols
        out = SubMatrix.empty(n0, n1, nat.MB_F64, self.buf.device)
        nat.check(rt.lib.mb_block_ger(rt.ctx, self.handle(), other.handle(), out.handle()))
        return out

    # ---- factorizations: the Breeze/LAPACK calls of DenseVecMatrix.luDecompose / choleskyDecompose / inverse ----
    def lu(self):
        """`brzLU(m)` (matrix/DenseVecMatrix.scala:302): (packed unit-lower L and U, permutation array with the
        reference's meaning: row i of L*U is row perm[i] of this block)."""
        rt = Runtime.get(); rt.sync_stream()
        out = self.copy()
        perm = (C.c_int32 * max(1, self._rows))()
        nat.check(rt.lib.mb_block_lu(rt.ctx, out.handle(), perm))
        return out, np.array(perm[: self._rows], dtype=np.int64)

    def cholesky(self) -> "SubMatrix":
        """`brzCholesky(m)` (:495,513): lower L with L L^T = this, zeros above the diagonal."""
        rt = Runtime.get(); rt.sync_stream()
        out = self.copy()
        nat.check(rt.lib.mb_block_cholesky(rt.ctx, out.handle()))
        return out

    def inverse(self) -> "SubMatrix":
        """`brzInv(m)` (:587,606)."""
        rt = Runtime.get(); rt.sync_stream()
        out = SubMatrix.empty(self._rows, self._cols, nat.MB_F64, self.buf.device)
        nat.check(rt.lib.mb_block_inverse(rt.ctx, self.handle(), out.handle()))
        return out

    def solveTriangular(self, rhs: "SubMatrix", lower: bool, unit: bool = False) -> "SubMatrix":
        """`this \\ rhs` for a triangular `this` (the `l \\ ...` of :364): returns X with this * X = rhs."""
        rt = Runtime.get(); rt.sync_stream()
        x = rhs.copy()
        nat.check(rt.lib.mb_block_trsm(rt.ctx, self.handle(), int(lower), int(unit), x.handle()))
        return x

    # ---- the local steps of DenseVecMatrix.computeSVD (matrix/DenseVecMatrix.scala:1464-1486, 1589-1606) ----
    def gramian(self) -> "SubMatrix":
        """This^T * this (n x n, exactly symmetric): the Gramian of computeGramianMatrix for the rows this block holds.
        A transposed view (a DenseVecMatrix row shard) is read in place."""
        rt = Runtime.get(); rt.sync_stream()
        out = SubMatrix.empty(self._cols, self._cols, nat.MB_F64, self.buf.device)
        nat.check(rt.lib.mb_block_gramian(rt.ctx, self.handle(), out.handle()))
        return out

    def symmetricEigen(self):
        """(w, V) of this symmetric block (lower triangle read): all eigenvalues as an ndarray ordered by |w| descending,
        the eigenvectors as the columns of an n x n block (parallel cyclic Jacobi on the device).  Raises MarlinError with
        code MB_ERR_NO_CONVERGENCE if the sweep cap is reached, where the reference's ARPACK path throws
        IllegalStateException."""
        rt = Runtime.get(); rt.sync_stream()
        n = self._rows
        V = SubMatrix.empty(n, n, nat.MB_F64, self.buf.device)
        w = (C.c_double * max(1, n))()
        sweeps = C.c_int32()
        nat.check(rt.lib.mb_block_syev(rt.ctx, self.handle(), V.handle(), w, C.byref(sweeps)))
        self.last_sweeps = int(sweeps.value)
        return np.array(w[:n], dtype=np.float64), V

    def add_(self, other: "SubMatrix") -> "SubMatrix":
        """In-place accumulate (the reduceByKey combine of BlockMatrix.scala:177 without a new allocation)."""
        rt = Runtime.get(); rt.sync_stream()
        nat.check(rt.lib.mb_block_add(rt.ctx, self.handle(), other.handle(), self.handle()))
        return self

    def transpose(self) -> "SubMatrix":
        """`denseBlock.t.copy` (matrix/BlockMatrix.scala:517): materialised transpose."""
        rt = Runtime.get(); rt.sync_stream()
        out = SubMatrix.empty(self._cols, self._rows, self.dtype, self.buf.device)
        nat.check(rt.lib.mb_block_transpose(rt.ctx, self.handle(), out.handle()))
        return out

    def copy(self, dtype: Optional[int] = None) -> "SubMatrix":
        """Breeze `.copy`: packed column-major copy of a view (optionally converting fp64 <-> bf16/fp32)."""
        rt = Runtime.get(); rt.sync_stream()
        out = SubMatrix.empty(self._rows, self._cols, self.dtype if dtype is None else dtype, self.buf.device)
        nat.check(rt.lib.mb_block_copy(rt.ctx, self.handle(), out.handle()))
        return out

    def assign(self, src: "SubMatrix") -> None:
        """`this(range) := src` — copy src into this view."""
        rt = Runtime.get(); rt.sync_stream()
        nat.check(rt.lib.mb_block_copy(rt.ctx, src.handle(), self.handle()))

    def sum(self) -> float:
        rt = Runtime.get(); rt.sync_stream()
        blk = self if self.dtype == nat.MB_F64 else self.copy(nat.MB_F64)
        out = C.c_double()
        nat.check(rt.lib.mb_block_sum(rt.ctx, blk.handle(), C.byref(out)))
        return float(out.value)

    # ---- host transfer (toBreeze / collect) ----
    @property
    def device(self):
        return self._sparse.values.device if self._sparse is not None else self.buf.device

    def toBreeze(self) -> np.ndarray:
        """Download as a (rows x cols) Fortran-ordered float64 ndarray (a sparse block through toDense)."""
        if self._rows == 0 or self._cols == 0:
            return np.zeros((self._rows, self._cols), order="F")
        if self._sparse is not None:
            return self.toDense().toBreeze()
        if self.buf.is_cuda:
            blk = self if (self.is_packed() and self.dtype == nat.MB_F64) else self.copy(nat.MB_F64)
            flat = blk.buf[: self._rows * self._cols].cpu().numpy()
            return flat.reshape((self._rows, self._cols), order="F")
        # host-resident block (CPU-side plumbing tests only): pure indexing, no arithmetic
        flat = self.buf.to(torch.float64).numpy()
        r = np.arange(self._rows)[:, None]
        c = np.arange(self._cols)[None, :]
        idx = self.offset + (c + r * self.ld if self.is_transpose else r + c * self.ld)
        return np.asfortranarray(flat[idx])

    to_numpy = toBreeze

    def __repr__(self):
        if self._sparse is not None:
            return f"SubMatrix({self._rows}x{self._cols}, sparse, nnz={self._sparse.nnz}, {self.device})"
        return f"SubMatrix({self._rows}x{self._cols}, ld={self.ld}, t={self.is_transpose}, {self.buf.dtype}, {self.buf.device})"


class RawBlock:
    """A column-major block at a raw device address that torch does not own — e.g. a staging slot in ANOTHER rank's HBM
    mapped through CUDA IPC.  Only usable as a GEMM output (`SubMatrix.multiply(..., out=RawBlock)`)."""

    def __init__(self, ptr: int, rows: int, cols: int, ld: int, dtype: int):
        self.ptr, self._rows, self._cols, self.ld, self._dtype = int(ptr), int(rows), int(cols), int(ld), int(dtype)
        self._handle = None

    @property
    def rows(self) -> int:
        return self._rows

    @property
    def cols(self) -> int:
        return self._cols

    @property
    def dtype(self) -> int:
        return self._dtype

    def slice(self, r0: int, r1: int, c0: int, c1: int) -> "RawBlock":
        esz = 8 if self._dtype == nat.MB_F64 else (4 if self._dtype == nat.MB_F32 else 2)
        return RawBlock(self.ptr + (r0 + c0 * self.ld) * esz, r1 - r0, c1 - c0, self.ld, self._dtype)

    def handle(self):
        if self._handle is None:
            rt = Runtime.get()
            h = nat.c_blk()
            nat.check(rt.lib.mb_block_wrap(rt.ctx, C.c_void_p(self.ptr), 0, self._rows, self._cols, self.ld, 0, self._dtype,
                                           C.byref(h)))
            self._handle = h
        return self._handle

    def __del__(self):
        h = getattr(self, "_handle", None)
        if h is not None:
            try:
                rt = Runtime._instance
                if rt is not None:
                    rt.lib.mb_block_free(rt.ctx, h)
            except Exception:
                pass

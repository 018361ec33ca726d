"""SparseVecMatrix — the drop-in for edu.nju.pasalab.marlin.matrix.SparseVecMatrix (matrix/SparseVecMatrix.scala).

An RDD[(Long, BSV[Double])] becomes, per rank, the rows this rank holds: int64 row `ids` (storage order) and one CSR
block of those rows on the device.  The block is the library's CSC handle of the transpose (mb_sparse with rows = nCols
and cols = the local row count), so its structure is checked by mb_sparse_check: column ids in [0, nCols), strictly
increasing within a row.  multiplySparse runs the row-wise SpGEMM of the library (mb_spvec_multiply).
"""
from __future__ import annotations

import ctypes as C
from typing import Tuple

import numpy as np
import torch

from .. import _native as nat
from ..runtime import Runtime, world
from .coordinate_matrix import CoordinateMatrix, _raise_gathered
from .dense_vec_matrix import DenseVecMatrix
from .sparse_matrix import SparseBlock
from .sub_matrix import SubMatrix

_ID_MAX = 2 ** 31 - 1


def _check_unique(ids: np.ndarray) -> None:
    srt = np.sort(ids)
    dup = np.flatnonzero(srt[1:] == srt[:-1])
    if len(dup):
        raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, f"SparseVecMatrix: repeated row id {srt[dup[0]]}")


def _download(h) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(rowptr, cols, values) of a library-owned row handle, which is then freed."""
    rt = Runtime.get()
    rows, cols, nnz = nat.c_i32(), nat.c_i32(), nat.c_i64()
    try:
        nat.check(rt.lib.mb_sparse_info(h, C.byref(rows), C.byref(cols), C.byref(nnz)))
        rp = np.empty(cols.value + 1, np.int32)
        ci = np.empty(max(nnz.value, 1), np.int32)
        va = np.empty(max(nnz.value, 1), np.float64)
        nat.check(rt.lib.mb_sparse_download(rt.ctx, h, rp.ctypes.data, ci.ctypes.data, va.ctypes.data))
    finally:
        rt.lib.mb_sparse_free(rt.ctx, h)
    return rp, ci[:nnz.value], va[:nnz.value]


class SparseVecMatrix:
    def __init__(self, rows=None, nRows: int = 0, nCols: int = 0):
        """rows: iterable of (id, SparseVector) held by THIS rank (the reference's RDD content), or a tuple of arrays
        (ids, rowptr, cols, values) of numpy arrays or lists.  nRows and nCols are the matrix's dimensions, as in the reference's constructor.
        Ids must lie in [0, nRows) and appear once; column ids must be sorted and distinct within a row (the reference
        accepts anything there and then sums repeated ids through reduceByKey)."""
        self.nRows, self.nCols = int(nRows), int(nCols)
        if isinstance(rows, tuple) and len(rows) == 4 and all(isinstance(a, (np.ndarray, list)) for a in rows):
            ids, rowptr, cols, vals = rows
        else:
            items = list(rows or [])
            ids = [int(i) for i, _ in items]
            lens = [len(v.indices) for _, v in items]
            rowptr = np.concatenate([[0], np.cumsum(lens, dtype=np.int64)])
            cols = np.concatenate([np.asarray(v.indices, np.int64) for _, v in items]) if items else np.zeros(0, np.int64)
            vals = np.concatenate([np.asarray(v.values, np.float64) for _, v in items]) if items else np.zeros(0)
        self.ids = np.asarray(ids, dtype=np.int64).reshape(-1)
        rowptr = np.asarray(rowptr, dtype=np.int64).reshape(-1)
        cols = np.asarray(cols, dtype=np.int64).reshape(-1)
        vals = np.asarray(vals, dtype=np.float64).reshape(-1)
        if self.nRows < 0 or self.nCols < 0 or self.nCols > _ID_MAX:
            raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, f"SparseVecMatrix: {self.nRows} x {self.nCols}")
        if len(self.ids) and (self.ids.min() < 0 or self.ids.max() > _ID_MAX):
            bad = self.ids[(self.ids < 0) | (self.ids > _ID_MAX)][0]
            raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, f"SparseVecMatrix: id {bad} is outside [0, 2147483647]")
        if len(self.ids) and self.ids.max() >= self.nRows:
            raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG,
                                          f"SparseVecMatrix: row id {self.ids.max()} is outside [0, {self.nRows})")
        _check_unique(self.ids)
        if rowptr.shape != (len(self.ids) + 1,) or rowptr[-1] != len(cols) or len(cols) != len(vals):
            raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, "SparseVecMatrix: rowptr, cols and values do not match")
        if len(cols) > _ID_MAX:
            raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, f"SparseVecMatrix: {len(cols)} non-zeros, at most 2^31 - 1")
        if len(cols) and (cols.min() < 0 or cols.max() >= max(self.nCols, 1)):
            raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, f"SparseVecMatrix: a column id is outside [0, {self.nCols})")
        self.block = SparseBlock.from_host(self.nCols, len(self.ids), rowptr, cols, vals)

    @classmethod
    def _from_block(cls, ids: np.ndarray, block: SparseBlock, nRows: int, nCols: int) -> "SparseVecMatrix":
        """A matrix over a device block the library wrote (trusted structure)."""
        m = cls.__new__(cls)
        m.nRows, m.nCols, m.ids, m.block = int(nRows), int(nCols), np.asarray(ids, np.int64), block
        return m

    # ------------------------------------------------------------------ host views
    def _host_rows(self):
        rp, ci, va = self.block.to_host()
        return self.ids, rp.astype(np.int64), ci.astype(np.int64), va

    def _gathered(self):
        """Every rank's (ids, rowptr, cols, values), in rank order."""
        rank, ws = world()
        if ws == 1:
            return [self._host_rows()]
        import torch.distributed as dist
        out = [None] * ws
        dist.all_gather_object(out, self._host_rows())
        return out

    def elementsCount(self) -> int:
        """:67-69 — rows.count(): the number of stored rows, not the number of non-zeros."""
        return sum(len(p[0]) for p in self._gathered_ids())      # object gather: works on NCCL-only groups too

    def toBreeze(self) -> np.ndarray:
        mat = np.zeros((self.nRows, self.nCols), order="F")
        for ids, rp, ci, va in self._gathered():
            r = np.repeat(ids, np.diff(rp))
            mat[r, ci] = va
        return mat

    # ------------------------------------------------------------------ multiplySparse (:22-50)
    def _all_rows_csr(self):
        """B laid out as one CSR over row ids [0, nRows) on this rank's device, absent ids empty: the row counts first
        (all_gather_object of ids and nnz), then the column and value buffers (all_gather of padded tensors)."""
        rt = Runtime.get()
        rank, ws = world()
        dev = rt.device
        own_rp = self.block.colptr.to(torch.int64)
        if ws == 1:
            pieces = [(self.ids, own_rp, self.block.rowidx, self.block.values)]
        else:
            import torch.distributed as dist
            meta = [None] * ws
            dist.all_gather_object(meta, (self.ids, int(self.block.nnz)))
            cpu = dist.get_backend() != "nccl"
            tdev = torch.device("cpu") if cpu else dev
            cap = max(1, max(n for _, n in meta))
            maxrows = max(len(i) for i, _ in meta) + 1

            def gather(t, n, dtype):
                buf = torch.zeros(n, dtype=dtype, device=tdev)
                buf[:t.numel()] = t.to(tdev)
                out = [torch.empty(n, dtype=dtype, device=tdev) for _ in range(ws)]
                dist.all_gather(out, buf)
                return out
            rps = gather(own_rp, maxrows, torch.int64)
            cis = gather(self.block.rowidx, cap, torch.int32)
            vas = gather(self.block.values, cap, torch.float64)
            pieces = [(ids, rps[r][:len(ids) + 1].to(dev), cis[r][:n].to(dev), vas[r][:n].to(dev))
                      for r, (ids, n) in enumerate(meta)]
        _check_unique(np.concatenate([p[0] for p in pieces]))        # the same ids, so the same error, on every rank
        counts = torch.zeros(self.nRows + 1, dtype=torch.int64, device=dev)
        for ids, rp, _, _ in pieces:
            if len(ids):
                counts[torch.from_numpy(ids + 1).to(dev)] = rp[1:] - rp[:-1]
        rowptr = torch.cumsum(counts, 0)
        nnz = int(rowptr[-1].item())
        cols = torch.empty(nnz, dtype=torch.int32, device=dev)
        vals = torch.empty(nnz, dtype=torch.float64, device=dev)
        for ids, rp, ci, va in pieces:
            if ci.numel():
                lens = rp[1:] - rp[:-1]
                local_row = torch.repeat_interleave(torch.arange(len(ids), device=dev), lens)
                start = rowptr[torch.from_numpy(ids).to(dev)]
                dest = start[local_row] + torch.arange(ci.numel(), device=dev) - rp[local_row]
                cols[dest] = ci
                vals[dest] = va
        return SparseBlock(self.nCols, self.nRows, rowptr.to(torch.int32), cols, vals)

    def multiplySparse(self, other: "SparseVecMatrix") -> CoordinateMatrix:
        """C = this * other as a CoordinateMatrix(entries, this.nRows, other.nCols) of float32 values.  Each rank
        multiplies its own rows against all of `other`, whose rows are gathered to every rank first.  Every stored value
        is rounded to float32, the products are float32, and C(i, j) sums them in A's stored order (k ascending) from the
        first product; an entry exists wherever some k is stored on both sides, zeros and cancellations included.  The
        result is bit-identical whatever the number of ranks.  this.nCols != other.nRows is a dimension mismatch (the
        reference silently drops the unmatched k)."""
        # the checks see the same values on every rank, so every rank raises before any rank enters the exchange
        if self.nCols != other.nRows:
            raise nat.MarlinArgumentError(nat.MB_ERR_DIM_MISMATCH, f"multiplySparse: this.nCols {self.nCols} does not "
                                          f"match other.nRows {other.nRows}")
        _check_unique(np.concatenate([p[0] for p in self._gathered_ids()]))
        B = other._all_rows_csr()
        rt = Runtime.get()
        rt.sync_stream()
        out = nat.c_sp()
        result = {}

        def run():
            nat.check(rt.lib.mb_spvec_multiply(rt.ctx, self.block.handle(), B.handle(), C.byref(out)))
            result["csr"] = _download(out)
        _raise_gathered(run)
        rp, ci, va = result["csr"]
        rows = np.repeat(self.ids, np.diff(rp))
        return CoordinateMatrix((rows, ci.astype(np.int64), va.astype(np.float32)), self.nRows, other.nCols)

    # ------------------------------------------------------------------ toDenseVecMatrix (:56-65)
    def toDenseVecMatrix(self) -> DenseVecMatrix:
        """Every row id in [0, nRows) exactly once across the ranks: each rank densifies its own rows on the device
        (mb_sparse_to_dense into the transposed view of the row-major shard) and takes a contiguous share of the ids no
        rank holds as zero rows.  A stored -0.0 stays -0.0; the reference adds the sparse row to a zero row, which gives
        +0.0."""
        rank, ws = world()
        held = np.concatenate([p[0] for p in self._gathered_ids()])
        missing = np.setdiff1d(np.arange(self.nRows, dtype=np.int64), held)
        lo, hi = (rank * len(missing)) // ws, ((rank + 1) * len(missing)) // ws
        ids = np.concatenate([self.ids, missing[lo:hi]])
        n, nloc = self.nCols, len(self.ids)
        if not len(ids):
            return DenseVecMatrix([], self.nRows, n)
        rt = Runtime.get()
        buf = torch.zeros(len(ids) * n, dtype=torch.float64, device=rt.device)
        data = SubMatrix(buf=buf, rows=len(ids), cols=n, ld=max(1, n), is_transpose=True)
        if nloc and n:
            own = data.slice(0, nloc, 0, n).t                  # held: its handle must outlive the call
            rt.sync_stream()
            nat.check(rt.lib.mb_sparse_to_dense(rt.ctx, self.block.handle(), own.handle()))
        return DenseVecMatrix(nRows=self.nRows, nCols=n, ids=ids, data=data)

    def _gathered_ids(self):
        rank, ws = world()
        if ws == 1:
            return [(self.ids,)]
        import torch.distributed as dist
        out = [None] * ws
        dist.all_gather_object(out, (self.ids,))
        return out

    # ------------------------------------------------------------------ DenseVecMatrix.toSparseVecMatrix
    @staticmethod
    def _from_dense(mat: DenseVecMatrix) -> "SparseVecMatrix":
        """DenseVecMatrix.scala:1333-1353 on the device (mb_dense_rows_to_sparse): the entries != 0.0 of each row in column
        order (NaN kept, +-0.0 dropped), vectors of length nCols (the reference gives them length nnz)."""
        m, n = mat.numRows(), mat.numCols()
        if mat.data is None or not len(mat.ids):
            return SparseVecMatrix((np.zeros(0, np.int64), np.zeros(1, np.int64), np.zeros(0, np.int64), np.zeros(0)), m, n)
        rt = Runtime.get()
        rt.sync_stream()
        h = nat.c_sp()
        nat.check(rt.lib.mb_dense_rows_to_sparse(rt.ctx, mat.data.handle(), C.byref(h)))
        rp, ci, va = _download(h)
        return SparseVecMatrix((mat.ids, rp, ci, va), m, n)


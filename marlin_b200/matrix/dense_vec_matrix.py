"""DenseVecMatrix — the drop-in for edu.nju.pasalab.marlin.matrix.DenseVecMatrix (matrix/DenseVecMatrix.scala)
on the hot path (the four multiply paths, toBlocks/toBlockMatrix, transpose, add).

An RDD[(Long, BDV[Double])] becomes a row shard per rank: `ids` (the row indices this rank holds, in
storage order, host side) and `data`, one device buffer of shape (len(ids) x numCols) in ROW-major
order — i.e. a transposed SubMatrix view, which is exactly what the reference builds per partition
before its dgemm (`rowsMat(::, i) := row_i`, DenseVecMatrix.scala:1670-1675).
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

from .. import _native as nat
from .. import comm
from ..runtime import Runtime, world
from .block import BlockID
from .distributed_matrix import DistributedMatrix
from .sub_matrix import SubMatrix


# the SparkConf keys the reference reads for its block algorithms (matrix/DenseVecMatrix.scala:313,499,591)
conf: Dict[str, int] = {"marlin.lu.basesize": 1000, "marlin.cholesky.basesize": 1000, "marlin.inverse.basesize": 1000}


def _ceil_len(total: int, parts: int) -> int:
    return int(math.ceil(float(total) / float(parts)))


def _runs(ids: np.ndarray) -> List[Tuple[int, int, int]]:
    """Maximal runs (pos0, id0, length) of rows whose ids are consecutive in storage order."""
    out = []
    n = len(ids)
    p = 0
    while p < n:
        q = p + 1
        while q < n and ids[q] == ids[q - 1] + 1:
            q += 1
        out.append((p, int(ids[p]), q - p))
        p = q
    return out


class DenseVecMatrix(DistributedMatrix):
    def __init__(self, rows=None, nRows: int = 0, nCols: int = 0, *, ids: Optional[np.ndarray] = None,
                 data: Optional[SubMatrix] = None, device=None):
        """rows: iterable of (index, vector) pairs held by THIS rank (the reference's RDD content), or pass
        ids + data (a row-major shard already on the device)."""
        self._nRows, self._nCols = int(nRows), int(nCols)
        if data is not None:
            self.ids = np.asarray(ids, dtype=np.int64)
            self.data = data
        else:
            pairs = [(int(i), np.asarray(v, dtype=np.float64)) for i, v in (rows or [])]
            self.ids = np.array([i for i, _ in pairs], dtype=np.int64)
            if pairs:
                host = np.ascontiguousarray(np.stack([v for _, v in pairs]))          # (local_rows x cols) row-major
                if device is None:
                    device = Runtime.get().device if Runtime.available() else torch.device("cpu")
                buf = torch.from_numpy(host.reshape(-1)).to(device)
                self.data = SubMatrix(buf=buf, rows=host.shape[0], cols=host.shape[1], ld=max(1, host.shape[1]),
                                      is_transpose=True)
            else:
                self.data = None

    # ------------------------------------------------------------------ dims (:55-69)
    def _gather(self, items: list) -> list:
        rank, ws = world()
        if ws == 1:
            return items
        import torch.distributed as dist
        out = [None] * ws
        dist.all_gather_object(out, items)
        return [x for part in out for x in part]

    def numCols(self) -> int:
        if self._nCols <= 0:
            vals = self._gather([self.data.cols] if self.data is not None and len(self.ids) else [])
            if not vals:
                raise nat.MarlinError(nat.MB_ERR_EMPTY, "empty collection")       # rows.first() on an empty RDD
            self._nCols = int(vals[0])
        return self._nCols

    def numRows(self) -> int:
        if self._nRows <= 0:
            vals = self._gather([int(self.ids.max())] if len(self.ids) else [])
            if not vals:
                raise nat.MarlinError(nat.MB_ERR_EMPTY, "empty collection")       # reduce on an empty RDD
            self._nRows = max(vals) + 1
        return self._nRows

    @property
    def getRows(self):
        return self.ids, self.data

    def toBreeze(self) -> np.ndarray:
        """:74-84"""
        m, n = self.numRows(), self.numCols()
        local = (self.ids, self.data.toBreeze()) if self.data is not None and len(self.ids) else (self.ids, np.zeros((0, n)))
        mat = np.zeros((m, n), order="F")
        for ids, arr in self._gather([local]):
            if len(ids):
                mat[ids, :] = arr
        return mat

    # ------------------------------------------------------------------ multiply overloads
    def multiply(self, other, *args, **kwargs):
        """multiply(other, cores) :103; multiply(other, splitMode) :109; multiply(other, cores, thr) :196;
        multiply(B: BDM[Double]) :1660; multiply(b: Double) :853"""
        from .distributed_vector import DistributedVector
        if isinstance(other, (int, float)) and not args:
            return self._scalar("multiply", float(other))
        if isinstance(other, DistributedVector):
            # multiply(vector: DistributedVector, splitMode: (Int, Int)) :149-154
            mode = args[0] if args else kwargs["splitMode"]
            if self.numCols() != other.length:
                raise nat.MarlinArgumentError(nat.MB_ERR_DIM_MISMATCH, "Dimension mismatch during matrix-matrix multiplication: "
                                              f"{self.numCols()} vs {other.length}")
            return self.toBlockMatrix(int(mode[0]), int(mode[1])).multiply(other)
        if isinstance(other, np.ndarray) and other.ndim == 1:
            if args or "splitMode" in kwargs:
                # multiply(vector: BDV[Double], splitMode: Int) :162-165
                return self.toBlockMatrix(int(args[0] if args else kwargs["splitMode"]), 1).multiply(other)
            return self._multiply_vector_local(other)                     # multiply(vector: BDV[Double]) :171-184
        if isinstance(other, (np.ndarray, SubMatrix)):
            return self._multiply_local(other)
        if args and isinstance(args[0], (tuple, list)):
            return self._multiply_split(other, tuple(args[0]))
        if "splitMode" in kwargs:
            return self._multiply_split(other, tuple(kwargs["splitMode"]))
        if args or "cores" in kwargs:
            cores = args[0] if args else kwargs["cores"]
            thr = args[1] if len(args) > 1 else kwargs.get("broadcastThreshold", 300)
            return self._multiply_auto(other, int(cores), int(thr))
        raise TypeError("multiply(DistributedMatrix) needs `cores` or a splitMode, as in the reference API")

    def _multiply_auto(self, other, cores: int, broadcastThreshold: int = 300):
        """:196-231"""
        from .block_matrix import BlockMatrix
        if self.numCols() != other.numRows():
            raise nat.MarlinArgumentError(nat.MB_ERR_DIM_MISMATCH, "Dimension mismatch during matrix-matrix multiplication: "
                                          f"{self.numCols()} vs {other.numRows()}")
        import ctypes as C
        lib = nat.load()
        strat = C.c_int32()
        mkn = (C.c_int32 * 3)()
        nat.check(lib.mb_choose_strategy(self.numRows(), self.numCols(), other.numCols(), cores, broadcastThreshold,
                                         int(isinstance(other, BlockMatrix)), C.byref(strat), mkn))
        if strat.value == 0:
            return self._multiply_local(other.toBreeze())                        # :204-205 / :221-222
        if strat.value == 1:
            if isinstance(other, DenseVecMatrix):
                # reference quirk (:206-207): that.multiply(this.toBreeze()) evaluates B * A_local
                return other._multiply_local(self.toBreeze())
            return other.multiplyBy(self.toBreeze())                             # :223-224
        return self._multiply_split(other, (mkn[0], mkn[1], mkn[2]))

    def _multiply_split(self, other, splitMode: Tuple[int, int, int]):
        """:109-141 — rows -> (m,k) / (k,n) block grids with the seq replication of toBlocks, then the
        m*k*n block products and the k-way sum (done by BlockMatrix._multiply_same_grid)."""
        from .block_matrix import BlockMatrix
        if self.numCols() != other.numRows():
            raise nat.MarlinArgumentError(nat.MB_ERR_DIM_MISMATCH, "Dimension mismatch during matrix-matrix multiplication: "
                                          f"{self.numCols()} vs {other.numRows()}")
        m, k, n = splitMode
        if not (m > 0 and k > 0 and n > 0):
            raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, f"not supported (m, k, n): ({m}, {k}, {n})")
        if isinstance(other, BlockMatrix):
            # :136-139 re-grids `that` with (m, k) rather than (k, n) — the reference's behaviour, kept
            return self.toBlockMatrix(m, k).multiply(other.toBlockMatrix(m, k))
        res = self.toBlockMatrix(m, k).multiply(other.toBlockMatrix(k, n))
        # the reference labels the result grid (m, n) as requested (:134)
        return res

    def _multiply_vector_local(self, vector: np.ndarray) -> np.ndarray:
        """multiply(vector: BDV[Double]): BDV[Double] :171-184 — every row dotted with the broadcast vector, collected
        into a local vector indexed by row id.  One gemv over the row-major shard (each row read once)."""
        vector = np.asarray(vector, dtype=np.float64).reshape(-1)
        parts = []
        if self.data is not None and len(self.ids):
            if self.data.cols != vector.shape[0]:
                raise nat.MarlinArgumentError(nat.MB_ERR_DIM_MISMATCH, "Dimension mismatch during matrix-vector multiplication: "
                                              f"{self.data.cols} vs {vector.shape[0]}")
            y = self.data.multiply(SubMatrix(vector.reshape(-1, 1), device=self.data.buf.device))
            parts = [(self.ids, y.toBreeze().reshape(-1))]
        parts = self._gather(parts)
        total = int(sum(len(i) for i, _ in parts))
        out = np.zeros(total)
        for ids, vals in parts:
            out[ids] = vals                                               # result(id) = v   (:181-183)
        return out

    def _multiply_local(self, B) -> "DenseVecMatrix":
        """multiply(B: BDM[Double]) :1660-1680 — B replicated on every rank (sc.broadcast), one GEMM per row shard,
        C rows keep the ids of A rows."""
        Bd = B if isinstance(B, SubMatrix) else None
        b_rows = Bd.rows if Bd is not None else B.shape[0]
        b_cols = Bd.cols if Bd is not None else B.shape[1]
        if self.numCols() != b_rows:
            raise nat.MarlinArgumentError(nat.MB_ERR_DIM_MISMATCH, "Dimension mismatch during matrix-matrix multiplication: "
                                          f"{self.numCols()} vs {b_rows}")
        if self.data is None or not len(self.ids):
            return DenseVecMatrix(ids=self.ids, data=self.data, nRows=0, nCols=b_cols)
        if Bd is None:
            Bd = SubMatrix(B, device=self.data.buf.device)
        nloc = self.data.rows
        out_dt = nat.MB_F32 if self.data.dtype == nat.MB_BF16 else self.data.dtype
        cbuf = torch.empty(nloc * b_cols, dtype=torch.float64 if out_dt == nat.MB_F64 else torch.float32,
                           device=self.data.buf.device)
        cshard = SubMatrix(buf=cbuf, rows=nloc, cols=b_cols, ld=max(1, b_cols), is_transpose=True)
        self.data.multiply(Bd, out=cshard)
        return DenseVecMatrix(ids=self.ids, data=cshard, nRows=0, nCols=b_cols)

    # ------------------------------------------------------------------ LU / Cholesky / inverse (:271-764)
    def _square_blocks(self, base: int):
        """All blocks of the ceil(n / base)^2 grid as device blocks on THIS rank (every rank factorises a replica)."""
        from . import factorizations as fz
        n = self.numRows()
        nb, sub = fz.grid(n, base)
        host = self.toBreeze()
        rt = Runtime.get()
        blocks = {(r, c): SubMatrix(host[r * sub:min(n, (r + 1) * sub), c * sub:min(n, (c + 1) * sub)], device=rt.device)
                  for r in range(nb) for c in range(nb)}
        return blocks, nb, sub, n

    def _finish(self, blocks, nb: int, n: int):
        from . import factorizations as fz
        from .block_matrix import BlockMatrix
        rank, ws = world()
        owner = lambda r, c: comm.elem_owner(r, c, nb, ws)
        return BlockMatrix(fz.block_pairs(blocks, owner, rank), n, n, nb, nb)

    def luDecompose(self, mode: str = "auto", baseSize: Optional[int] = None, keepUnfactoredDiagonal: bool = False):
        """luDecompose(mode) :283-466 -> (BlockMatrix holding L (unit lower) and U packed, permutation array: row i of
        L*U is row perm[i] of this matrix).  Deviation, on purpose: the reference stores the ORIGINAL diagonal block for
        every block row but the last (`scatterRdds(i)(0) = matFirst.cache()`, :355), which makes P A = L U false;
        `keepUnfactoredDiagonal=True` reproduces that, the default stores the factors."""
        from . import factorizations as fz
        if self.numRows() != self.numCols():
            raise nat.MarlinArgumentError(nat.MB_ERR_DIM_MISMATCH, f"LU decompose only support square matrix: {self.numRows()} v.s {self.numCols()}")
        n = self.numRows()
        if not fz.mode_is_dist(mode, n):
            blocks, _, _, _ = self._square_blocks(n)
            packed, perm = blocks[(0, 0)].lu()
            return self._finish({(0, 0): packed}, 1, n), [int(p) for p in perm]
        blocks, nb, sub, n = self._square_blocks(baseSize or conf.get("marlin.lu.basesize", 1000))
        out, p_array = fz.lu_blocks(blocks, nb, sub, n, keepUnfactoredDiagonal)
        return self._finish(out, nb, n), p_array

    def choleskyDecompose(self, mode: str = "auto", baseSize: Optional[int] = None):
        """choleskyDecompose(mode) :475-561 -> BlockMatrix of the lower-triangular blocks of L, L L^T = this (no blocks
        above the diagonal, as in the reference; dims are set explicitly where the reference leaves them to be inferred)."""
        from . import factorizations as fz
        if self.numRows() != self.numCols():
            raise nat.MarlinArgumentError(nat.MB_ERR_DIM_MISMATCH, f"LU decompose only support square matrix: {self.numRows()} v.s {self.numCols()}")
        n = self.numRows()
        if not fz.mode_is_dist(mode, n):
            blocks, _, _, _ = self._square_blocks(n)
            return self._finish({(0, 0): blocks[(0, 0)].cholesky()}, 1, n)
        blocks, nb, _, n = self._square_blocks(baseSize or conf.get("marlin.cholesky.basesize", 1000))
        return self._finish(fz.cholesky_blocks({k: v for k, v in blocks.items() if k[0] >= k[1]}, nb), nb, n)

    def inverse(self, mode: str = "auto", baseSize: Optional[int] = None):
        """inverse() :271-273, inverse(mode) :568-764"""
        from . import factorizations as fz
        if self.numRows() != self.numCols():
            raise nat.MarlinArgumentError(nat.MB_ERR_DIM_MISMATCH, f"Inversion only support square matrix: {self.numRows()} v.s {self.numCols()}")
        n = self.numRows()
        if not fz.mode_is_dist(mode, n):
            blocks, _, _, _ = self._square_blocks(n)
            return self._finish({(0, 0): blocks[(0, 0)].inverse()}, 1, n)
        blocks, nb, _, n = self._square_blocks(baseSize or conf.get("marlin.inverse.basesize", 1000))
        return self._finish(fz.inverse_blocks(blocks, nb), nb, n)

    # ------------------------------------------------------------------ SVD (:1464-1652)
    def computeSVD(self, k: int, computeU: bool = False, rCond: float = 1e-9, mode: str = "auto"):
        """computeSVD(k, computeU, rCond) :1531-1541 and the private mode overload :1557-1652 ->
        (U: DenseVecMatrix or None, s: ndarray of the sk leading singular values, V: ndarray n x sk).

        mode is chosen and validated exactly as in the reference (mb_svd_mode: "auto", "local-svd", "local-eigs",
        "dist-eigs", with its `require` messages).  Deliberate deviations, on every mode:
          * one Gramian G = A^T A on the device (split-K DMMA, summed in a fixed order) and one full eigendecomposition
            of G by parallel Jacobi; "dist-eigs" exists in the reference to keep n^2 doubles off the driver.  Device
            memory, not the 65535-column cap, bounds n: G, V and the eigensolver's four working copies take about
            48 * n^2 bytes besides A (about n = 40000 on an 80 GB H100; beyond that MarlinError MB_ERR_OOM).  Unlike
            ARPACK the result never has fewer than k values;
          * the Gramian's summation order differs from the reference's row-by-row dspr, so the results agree with it
            within rounding, not bitwise;
          * s = sqrt(|w|), the singular values of G as local-svd (dgesdd) returns them.
        With several ranks every rank forms the Gramian of its rows (zeros if it holds none); the partials are exchanged
        and summed in rank order on every rank, so all ranks hold the same G bit for bit and compute the same s and V.
        The rows of U stay on the rank that holds the matching rows of this matrix."""
        import ctypes as C
        lib = nat.load()
        n = self.numCols()
        cm = C.c_int32()
        nat.check(lib.mb_svd_mode(n, int(k), str(mode).encode(), C.byref(cm)))
        rank, ws = world()
        dev = self.data.buf.device if self.data is not None else Runtime.get().device
        if self.data is not None and len(self.ids):
            g = self.data.gramian()
        else:
            g = SubMatrix.zeros(n, n, nat.MB_F64, dev)
        if ws > 1:
            sends = [(src, dst, ("gram", src)) for src in range(ws) for dst in range(ws) if src != dst]
            got = comm.exchange(sends, {("gram", rank): g.buf[: n * n]},
                                lambda key: torch.empty(n * n, dtype=torch.float64, device=dev), rank)
            parts = [g if r == rank else SubMatrix(buf=got[("gram", r)], rows=n, cols=n, ld=n) for r in range(ws)]
            g = parts[0]
            for p in parts[1:]:
                g = g.add(p)
        w, vblk = g.symmetricEigen()
        sigmas = np.sqrt(np.abs(w))
        sk = lib.mb_svd_rank(sigmas.ctypes.data_as(nat.c_dp), n, int(k), float(rCond))
        if sk < 0:
            nat.check(sk)
        s = sigmas[:sk].copy()
        V = vblk.slice(0, n, 0, sk).toBreeze() if sk else np.zeros((n, 0), order="F")
        if not computeU:
            return None, s, V
        # N = V_k * S_k^-1 (:1635-1646), column j divided by sigma_j, then U = this.multiply(N) (:1647)
        nmat = SubMatrix.empty(n, sk, nat.MB_F64, dev)
        for j in range(sk):
            vblk.slice(0, n, j, j + 1)._divide_into(float(sigmas[j]), nmat.slice(0, n, j, j + 1))
        return self._multiply_local(nmat), s, V

    # ------------------------------------------------------------------ element-wise (:771-871)
    def _scalar(self, op: str, b: float) -> "DenseVecMatrix":
        if self.data is None:
            return self
        f = {"add": lambda s: s.add(b), "subtract": lambda s: s.subtract(b), "multiply": lambda s: s.multiply(b),
             "divide": lambda s: s.divide(b), "subtractBy": lambda s: s.subtractBy(b), "divideBy": lambda s: s.divideBy(b)}[op]
        return DenseVecMatrix(ids=self.ids, data=f(self.data), nRows=self.numRows(), nCols=self.numCols())

    def _binary(self, other, op: str) -> "DenseVecMatrix":
        from .block_matrix import BlockMatrix
        if isinstance(other, (int, float)):
            return self._scalar(op, float(other))
        if isinstance(other, BlockMatrix):
            other = other.toDenseVecMatrix()                                     # :782-783
        if not isinstance(other, DenseVecMatrix):
            raise nat.MarlinArgumentError(nat.MB_ERR_UNSUPPORTED, f"Do not support this type {type(other)} for {op} operation")
        if self.numRows() != other.numRows() or self.numCols() != other.numCols():
            raise nat.MarlinArgumentError(nat.MB_ERR_DIM_MISMATCH, f"Dimension mismatch: {self.numRows()}x{self.numCols()} vs "
                                          f"{other.numRows()}x{other.numCols()}")
        # rows.join(that.rows) (:777-780) is an INNER join: a row id present on one side only is dropped from the result
        theirs = set(int(i) for part in self._gather([other.ids.tolist()]) for i in part)
        keep = [p for p, i in enumerate(self.ids) if int(i) in theirs]
        me = self if len(keep) == len(self.ids) else self._select_rows(keep)
        if me.data is None or not len(me.ids):
            other._aligned_to(me)                                                # still collective on every rank
            return DenseVecMatrix(ids=me.ids, data=me.data, nRows=self.numRows(), nCols=self.numCols())
        other = other._aligned_to(me)
        fn = {"add": SubMatrix.add, "subtract": SubMatrix.subtract, "dotProduct": SubMatrix.elementMultiply}[op]
        return DenseVecMatrix(ids=me.ids, data=fn(me.data, other.data), nRows=self.numRows(), nCols=self.numCols())

    def _select_rows(self, positions) -> "DenseVecMatrix":
        """The local rows at `positions` (ascending local order) as a new packed row-major shard."""
        nc = self.numCols()
        ids = self.ids[list(positions)] if len(positions) else np.zeros(0, dtype=np.int64)
        if not len(positions):
            empty = SubMatrix(buf=torch.zeros(0, dtype=self.data.buf.dtype, device=self.data.buf.device), rows=0, cols=nc,
                              ld=max(1, nc), is_transpose=True)
            return DenseVecMatrix(ids=ids, data=empty, nRows=self._nRows, nCols=nc)
        buf = torch.empty(len(positions) * nc, dtype=self.data.buf.dtype, device=self.data.buf.device)
        shard = SubMatrix(buf=buf, rows=len(positions), cols=nc, ld=max(1, nc), is_transpose=True)
        # runs of consecutive positions move as one strided copy
        p = 0
        while p < len(positions):
            q = p
            while q + 1 < len(positions) and positions[q + 1] == positions[q] + 1:
                q += 1
            shard.slice(p, q + 1, 0, nc).assign(self.data.slice(positions[p], positions[q] + 1, 0, nc))
            p = q + 1
        return DenseVecMatrix(ids=ids, data=shard, nRows=self._nRows, nCols=nc)

    def _aligned_to(self, ref: "DenseVecMatrix") -> "DenseVecMatrix":
        """Re-shard / re-order rows so that they line up with `ref`'s ids (the join on row index)."""
        rank, ws = world()
        if ws == 1 and np.array_equal(self.ids, ref.ids):
            return self
        return _redistribute_rows(self, ref.ids, self._gather([(rank, ref.ids)]))

    def add(self, other):
        """add(other: DistributedMatrix) :771-788, add(b: Double) :817-822"""
        return self._binary(other, "add")

    def subtract(self, other):
        """:795-834"""
        return self._binary(other, "subtract")

    def dotProduct(self, other):
        return self._binary(other, "dotProduct")

    def divide(self, b: float):
        """:866-871"""
        return self._scalar("divide", float(b))

    def subtractBy(self, b: float):
        return self._scalar("subtractBy", float(b))

    def divideBy(self, b: float):
        return self._scalar("divideBy", float(b))

    def sum(self) -> float:
        parts = self._gather([self.data.sum()] if self.data is not None and len(self.ids) else [])
        if not parts:
            raise nat.MarlinError(nat.MB_ERR_EMPTY, "empty collection")
        total = 0.0
        for p in parts:
            total += p
        return total

    # ------------------------------------------------------------------ transpose (:1420-1436)
    def transpose(self, numBlocks: Optional[int] = None):
        """toBlockMatrix(min(parallelism, rows/2), 1).transpose(); parallelism defaults to the number of GPUs
        (spark.default.parallelism), or 2 on one GPU to match the reference suite's local[2]."""
        rank, ws = world()
        par = numBlocks if numBlocks is not None else (ws if ws > 1 else 2)
        return self.toBlockMatrix(min(par, self.numRows() // 2), 1).transpose()

    # ------------------------------------------------------------------ rows -> blocks (:1084-1328)
    def toBlockMatrix(self, numByRow: int, numByCol: int):
        """:1259-1328 — ceil-sized blocks; the strided `mat(r, ::) := vec.t` fills become strided device copies
        of whole row runs, and the groupByKey becomes one grouped exchange of the pieces that change GPU."""
        from .block_matrix import BlockMatrix
        mRows, mCols = self.numRows(), self.numCols()
        brs, bcs = _ceil_len(mRows, numByRow), _ceil_len(mCols, numByCol)
        by_row, by_col = int(math.ceil(mRows / brs)), int(math.ceil(mCols / bcs))
        rank, ws = world()
        owner = (lambda r, c: comm.elem_owner(r, c, by_col, ws)) if ws > 1 else (lambda r, c: 0)
        my_runs = []
        for pos0, id0, length in _runs(self.ids):
            # cut runs at block-row boundaries
            while length > 0:
                br = id0 // brs
                take = min(length, (br + 1) * brs - id0)
                my_runs.append((rank, pos0, id0, take))
                pos0 += take; id0 += take; length -= take
        all_runs = self._gather(my_runs)
        dt = self.data.buf.dtype if self.data is not None else torch.float64
        dev = self.data.buf.device if self.data is not None else (Runtime.get().device if Runtime.available() else torch.device("cpu"))
        mbdt = nat.MB_F64 if dt == torch.float64 else (nat.MB_BF16 if dt == torch.bfloat16 else nat.MB_F32)
        sends, send_bufs, pastes = [], {}, []
        for (src, pos0, id0, take) in all_runs:
            br = id0 // brs
            for bc in range(by_col):
                c0, c1 = bc * bcs, min((bc + 1) * bcs, mCols)
                dst = owner(br, bc)
                key = (src, id0, bc)
                piece = self.data.slice(pos0, pos0 + take, c0, c1) if src == rank else None
                if dst == rank:
                    pastes.append((key, (br, bc), id0 - br * brs, take, c1 - c0, piece))
                if src != dst:
                    sends.append((src, dst, key))
                    if src == rank:
                        packed = piece.copy()
                        send_bufs[key] = packed.buf[: packed.rows * packed.cols]
        shapes = {p[0]: (p[3], p[4]) for p in pastes}
        got = comm.exchange(sends, send_bufs, lambda key: torch.empty(shapes[key][0] * shapes[key][1], dtype=dt, device=dev),
                            rank) if ws > 1 else {}
        blocks: Dict[Tuple[int, int], SubMatrix] = {}
        for key, (br, bc), r0, take, width, piece in pastes:
            if (br, bc) not in blocks:
                rows = mRows - br * brs if br * brs + brs - 1 >= mRows else brs
                cols = mCols - bc * bcs if bc * bcs + bcs - 1 >= mCols else bcs
                blocks[(br, bc)] = SubMatrix.zeros(rows, cols, mbdt, dev)       # BDM.zeros (:1318)
            if piece is None:
                piece = SubMatrix(buf=got[key], rows=take, cols=width, ld=max(1, take))
            blocks[(br, bc)].slice(r0, r0 + take, 0, width).assign(piece)
        res = [(BlockID(r, c), blk) for (r, c), blk in sorted(blocks.items())]
        return BlockMatrix(res, mRows, mCols, by_row, by_col)

    def toBlocks(self, m: int, k: int, n: int, mode: str):
        """:1084-1223 — the blocks of toBlockMatrix plus the seq replication keys; on GPUs the replicas are the
        tile transfers planned in marlin_b200.comm, so this returns (BlockID(row, col, seq), block) pairs that
        alias one device block per (row, col)."""
        mode = mode.lower()
        if mode not in ("right", "left"):
            raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, f"only 'right' mode or 'left' mode is supported, you should change mode {mode}")
        if not (m > 0 and k > 0 and n > 0):
            raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, f"not supported (m, k, n): ({m}, {k}, {n})")
        out = []
        if mode == "right":
            for b, mat in self.toBlockMatrix(m, k).blocks:
                for i in range(n):
                    out.append((BlockID(b.row, i, b.row * n * k + i * k + b.column), mat))     # :1115,:1151
        else:
            for b, mat in self.toBlockMatrix(k, n).blocks:
                for i in range(m):
                    out.append((BlockID(i, b.column, i * n * k + b.column * k + b.row), mat))  # :1182,:1217
        return out

    @staticmethod
    def _from_block_matrix(bm) -> "DenseVecMatrix":
        """BlockMatrix.toDenseVecMatrix (matrix/BlockMatrix.scala:575-594): rows of block-row r are assembled,
        row-major, on owner(r, 0)."""
        nr, nc = bm.numRows(), bm.numCols()
        rl, cl = _ceil_len(nr, bm.numBlksByRow()), _ceil_len(nc, bm.numBlksByCol())
        rank, ws = world()
        local = {(b.row, b.column): s for b, s in bm.blocks}
        dt = bm._local_dtype()
        dev = Runtime.get().device if Runtime.available() else torch.device("cpu")
        sends, send_bufs = [], {}
        my_rows = [r for r in range(bm.numBlksByRow()) if bm.owner(r, 0) == rank]
        for r in range(bm.numBlksByRow()):
            dst = bm.owner(r, 0)
            for c in range(bm.numBlksByCol()):
                src = bm.owner(r, c)
                if src != dst:
                    sends.append((src, dst, (r, c)))
                    if src == rank:
                        blk = local[(r, c)] if local[(r, c)].is_packed() else local[(r, c)].copy()
                        send_bufs[(r, c)] = blk.buf[: blk.rows * blk.cols]
        dims = lambda r, c: (min(rl, nr - r * rl), min(cl, nc - c * cl))
        got = comm.exchange(sends, send_bufs, lambda key: torch.empty(dims(*key)[0] * dims(*key)[1], dtype=dt, device=dev),
                            rank) if ws > 1 else {}
        nloc = sum(dims(r, 0)[0] for r in my_rows)
        ids = np.concatenate([np.arange(r * rl, r * rl + dims(r, 0)[0], dtype=np.int64) for r in my_rows]) if my_rows \
            else np.zeros(0, dtype=np.int64)
        if nloc == 0:
            return DenseVecMatrix(ids=ids, data=None, nRows=nr, nCols=nc)
        buf = torch.zeros(nloc * nc, dtype=dt, device=dev)                        # BDV.zeros (:587)
        shard = SubMatrix(buf=buf, rows=nloc, cols=nc, ld=max(1, nc), is_transpose=True)
        off = 0
        for r in my_rows:
            rows = dims(r, 0)[0]
            for c in range(bm.numBlksByCol()):
                if (r, c) in local:
                    src = local[(r, c)]
                else:
                    rr, cc = dims(r, c)
                    src = SubMatrix(buf=got[(r, c)], rows=rr, cols=cc, ld=max(1, rr))
                shard.slice(off, off + rows, c * cl, c * cl + src.cols).assign(src)
            off += rows
        return DenseVecMatrix(ids=ids, data=shard, nRows=nr, nCols=nc)

    # ------------------------------------------------------------------ I/O (next-row (f)-3)
    def _save_rows(self, path: str) -> None:
        import os
        from ..utils.mt_utils import _jdouble
        rank, ws = world()
        os.makedirs(path, exist_ok=True)
        arr = self.data.toBreeze() if self.data is not None and len(self.ids) else np.zeros((0, 0))
        with open(os.path.join(path, f"part-{rank:05d}"), "w") as fh:
            for pos, idx in enumerate(self.ids):
                fh.write(f"{int(idx)}:DenseVector(" + ", ".join(_jdouble(v) for v in arr[pos, :]) + ")\n")

    def saveToFileSystem(self, path: str) -> None:
        """:1042-1046 — one line per row, `t._1 + ":" + t._2.toString`.  The row is a Breeze DenseVector, whose toString
        is `DenseVector(v0, v1, ...)`, so that is what the reference's files contain (its own loadMatrixFile cannot read
        them back; MTUtils.loadMatrixFile here accepts both this and the plain `index:v,v,...` form)."""
        self._save_rows(path)

    def saveWithDescription(self, path: str) -> None:
        """:1055-1064 — the rows as above plus `_description`: `MatrixName<TAB>N/A` / `MatrixSize<TAB>rows cols`."""
        import os
        self._save_rows(path)
        rows, cols = self.numRows(), self.numCols()
        if world()[0] == 0:
            with open(os.path.join(path, "_description"), "w") as fh:
                fh.write(f"MatrixName\tN/A\nMatrixSize\t{rows} {cols}")

    def print(self) -> None:
        arr = self.data.toBreeze() if self.data is not None else np.zeros((0, 0))
        for pos, idx in enumerate(self.ids[:20]):
            print(f"index: {int(idx)}, vector: {arr[pos, :8]}")


def _redistribute_rows(src: DenseVecMatrix, want_ids: np.ndarray, all_wants: list) -> DenseVecMatrix:
    """Row join: deliver to every rank the rows of `src` whose ids it lists in want_ids, in that order."""
    rank, ws = world()
    nc = src.numCols()
    have = src._gather([(rank, src.ids)])
    where: Dict[int, Tuple[int, int]] = {}
    for r, ids in have:
        for pos, i in enumerate(ids):
            where[int(i)] = (r, pos)
    dt = src.data.buf.dtype if src.data is not None else torch.float64
    dev = src.data.buf.device if src.data is not None else Runtime.get().device
    sends, send_bufs = [], {}
    local_copy = []
    for dst, ids in sorted(all_wants, key=lambda t: t[0]):
        for dpos, i in enumerate(ids):
            if int(i) not in where:
                continue                     # inner join: rows missing on one side are dropped
            s, spos = where[int(i)]
            if s == dst:
                if dst == rank:
                    local_copy.append((spos, dpos))
            else:
                sends.append((s, dst, (int(i),)))
                if s == rank:
                    send_bufs[(int(i),)] = src.data.slice(spos, spos + 1, 0, nc).copy().buf[:nc]
    got = comm.exchange(sends, send_bufs, lambda key: torch.empty(nc, dtype=dt, device=dev), rank) if ws > 1 else {}
    n = len(want_ids)
    buf = torch.zeros(n * nc, dtype=dt, device=dev)
    shard = SubMatrix(buf=buf, rows=n, cols=nc, ld=max(1, nc), is_transpose=True)
    for spos, dpos in local_copy:
        shard.slice(dpos, dpos + 1, 0, nc).assign(src.data.slice(spos, spos + 1, 0, nc))
    pos_of = {int(i): p for p, i in enumerate(want_ids)}
    for (i,), b in got.items():
        shard.slice(pos_of[i], pos_of[i] + 1, 0, nc).assign(SubMatrix(buf=b, rows=1, cols=nc, ld=1))
    return DenseVecMatrix(ids=np.asarray(want_ids, dtype=np.int64), data=shard, nRows=src.numRows(), nCols=nc)

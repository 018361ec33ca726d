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


# the stream of the Lanczos start vector: every rank starts from the same bits
EIGS_SEED = 1557


def symmetric_eigs(op, n: int, k: int, tol: float, max_iter: int):
    """EigenValueDecomposition.symmetricEigs (:1725-1834) on the device: the k largest-magnitude eigenpairs of the
    symmetric operator `op(x, y)` (writes y = Op x; both are mb_block handles of n x 1 device vectors), ncv =
    min(2k, n).  -> (eigenvalues descending, their eigenvectors as the columns of an n x k SubMatrix,
    {"applications": operator calls, "restarts": restarts taken})."""
    import ctypes as C
    rt = Runtime.get()
    rt.sync_stream()
    h = C.c_void_p()
    nat.check(rt.lib.mb_eigs_create(rt.ctx, n, k, min(2 * k, n), float(tol), int(max_iter), EIGS_SEED, C.byref(h)))
    try:
        ido, x, y = C.c_int32(0), nat.c_blk(), nat.c_blk()
        applications = 0
        while True:
            nat.check(rt.lib.mb_eigs_step(rt.ctx, h, C.byref(ido), C.byref(x), C.byref(y)))
            if ido.value == 99:
                break
            op(x, y)
            applications += 1
        w = np.zeros(k)
        Z = SubMatrix.empty(n, k, nat.MB_F64, rt.device)
        nconv, iters = C.c_int32(), C.c_int32()
        nat.check(rt.lib.mb_eigs_result(rt.ctx, h, w.ctypes.data_as(nat.c_dp), Z.handle(), C.byref(nconv), C.byref(iters)))
    finally:
        rt.lib.mb_eigs_destroy(h)
    return w, Z, {"applications": applications, "restarts": int(iters.value)}


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
        """All blocks of the ceil(n / base)^2 grid as device blocks on THIS rank ("breeze" mode: the whole matrix)."""
        from . import factorizations as fz
        n = self.numRows()
        nb, sub = fz.grid(n, base)
        host = self.toBreeze()
        rt = Runtime.get()
        blocks = {(r, c): SubMatrix(host[r * sub:min(n, (r + 1) * sub), c * sub:min(n, (c + 1) * sub)], device=rt.device)
                  for r in range(nb) for c in range(nb)}
        return blocks, nb, sub, n

    def _grid_blocks(self, nb: int, sub: int, want=lambda r, c: True):
        """The fp64 blocks (r, c) of the nb x nb grid (block length sub) that comm.elem_owner places on THIS rank and
        `want` keeps, built from the rows each rank holds: the pieces of one block row that change rank travel in one
        exchange, so no rank ever holds more than its own blocks and one block row of pieces."""
        n = self.numRows()
        rank, ws = world()
        dev = self.data.buf.device if self.data is not None else Runtime.get().device
        owner = lambda r, c: comm.elem_owner(r, c, nb, ws)
        size = lambda k: n - sub * (nb - 1) if k == nb - 1 else sub
        my_runs = []
        for pos0, id0, length in (_runs(self.ids) if self.data is not None else []):
            while length > 0:
                br = id0 // sub
                take = min(length, (br + 1) * sub - id0)
                my_runs.append((rank, pos0, id0, take))
                pos0 += take; id0 += take; length -= take
        all_runs = self._gather(my_runs)
        blocks = {(r, c): SubMatrix.zeros(size(r), size(c), nat.MB_F64, dev)       # BDM.zeros (:1318)
                  for r in range(nb) for c in range(nb) if owner(r, c) == rank and want(r, c)}
        for br in range(nb):
            sends, send_bufs, pastes = [], {}, []
            for (src, pos0, id0, take) in all_runs:
                if id0 // sub != br:
                    continue
                for bc in range(nb):
                    if not want(br, bc):
                        continue
                    dst, key = owner(br, bc), (src, id0, bc)
                    piece = self.data.slice(pos0, pos0 + take, bc * sub, bc * sub + size(bc)) if src == rank else None
                    if dst == rank:
                        pastes.append((key, bc, id0 - br * sub, take, piece))
                    elif src == rank:
                        send_bufs[key] = piece.copy(nat.MB_F64).buf
                    if src != dst:
                        sends.append((src, dst, key))
            got = comm.exchange(sends, send_bufs, lambda key: torch.empty(
                [p[3] for p in pastes if p[0] == key][0] * size(key[2]), dtype=torch.float64, device=dev), rank) if ws > 1 else {}
            del send_bufs
            for key, bc, r0, take, piece in pastes:
                if piece is None:
                    piece = SubMatrix(buf=got.pop(key), rows=take, cols=size(bc), ld=max(1, take))
                blocks[(br, bc)].slice(r0, r0 + take, 0, size(bc)).assign(piece)
        return blocks

    def _factor_dist(self, kind: str, base: int, keep_unfactored_diagonal: bool = False):
        """The sharded block algorithm: this rank's result blocks (and the pivot list for LU)."""
        from . import factorizations as fz
        n = self.numRows()
        nb, sub = fz.grid(n, base)
        rank, ws = world()
        dev = self.data.buf.device if self.data is not None else Runtime.get().device
        want = (lambda r, c: r >= c) if kind == "cholesky" else (lambda r, c: True)
        store = {("A", r, c): b for (r, c), b in self._grid_blocks(nb, sub, want).items()}
        del want
        pivots = {}
        fz.run(kind, store, nb, sub, n, rank, ws, dev, keep_unfactored_diagonal, pivots)
        if kind == "inverse":
            fz.run("inverse_back", store, nb, sub, n, rank, ws, dev)
            return {(r, c): b for (_, r, c), b in store.items()}, nb, n
        if kind == "lu":
            out, p_array = fz.finish_lu(store, pivots, nb, sub, n, rank, ws, dev)
            return out, nb, n, p_array
        return {(r, c): b for (_, r, c), b in store.items()}, nb, n

    def _finish(self, blocks, nb: int, n: int):
        """Blocks already on their owner (comm.elem_owner, MatrixElemOpPartitioner order) -> the result BlockMatrix."""
        from . import factorizations as fz
        from .block_matrix import BlockMatrix
        return BlockMatrix(fz.block_pairs(blocks), n, n, nb, nb, sparse=False)

    def luDecompose(self, mode: str = "auto", baseSize: Optional[int] = None, keepUnfactoredDiagonal: bool = False):
        """luDecompose(mode) :283-466 -> (BlockMatrix holding L (unit lower) and U packed, permutation array: row i of
        L*U is row perm[i] of this matrix).  Deviation, on purpose: the reference stores the ORIGINAL diagonal block for
        every block row but the last (`scatterRdds(i)(0) = matFirst.cache()`, :355), which makes P A = L U false;
        `keepUnfactoredDiagonal=True` reproduces that, the default stores the factors.  "dist" mode is sharded across
        the ranks (see matrix/factorizations.py): every rank gets the full permutation array."""
        from . import factorizations as fz
        if self.numRows() != self.numCols():
            raise nat.MarlinArgumentError(nat.MB_ERR_DIM_MISMATCH, f"LU decompose only support square matrix: {self.numRows()} v.s {self.numCols()}")
        n = self.numRows()
        if not fz.mode_is_dist(mode, n):
            blocks, _, _, _ = self._square_blocks(n)
            packed, perm = blocks[(0, 0)].lu()
            return self._finish_breeze({(0, 0): packed}, n), [int(p) for p in perm]
        out, nb, n, p_array = self._factor_dist("lu", baseSize or conf.get("marlin.lu.basesize", 1000), keepUnfactoredDiagonal)
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
            return self._finish_breeze({(0, 0): blocks[(0, 0)].cholesky()}, n)
        return self._finish(*self._factor_dist("cholesky", baseSize or conf.get("marlin.cholesky.basesize", 1000)))

    def inverse(self, mode: str = "auto", baseSize: Optional[int] = None):
        """inverse() :271-273, inverse(mode) :568-764"""
        from . import factorizations as fz
        if self.numRows() != self.numCols():
            raise nat.MarlinArgumentError(nat.MB_ERR_DIM_MISMATCH, f"Inversion only support square matrix: {self.numRows()} v.s {self.numCols()}")
        n = self.numRows()
        if not fz.mode_is_dist(mode, n):
            blocks, _, _, _ = self._square_blocks(n)
            return self._finish_breeze({(0, 0): blocks[(0, 0)].inverse()}, n)
        return self._finish(*self._factor_dist("inverse", baseSize or conf.get("marlin.inverse.basesize", 1000)))

    def _finish_breeze(self, blocks, n: int):
        """"breeze" mode: every rank computed the one block; rank 0 (its elem_owner) keeps it."""
        rank, _ = world()
        return self._finish(blocks if rank == 0 else {}, 1, n)

    # ------------------------------------------------------------------ SVD (:1464-1652)
    def computeSVD(self, k: int, computeU: bool = False, rCond: float = 1e-9, mode: str = "auto", *,
                   maxIter: Optional[int] = None, tol: Optional[float] = None):
        """computeSVD(k, computeU, rCond) :1531-1541 and the private mode overload :1557-1652 ->
        (U: DenseVecMatrix or None, s: ndarray of the sk leading singular values, V: ndarray n x sk).

        Without maxIter and tol, mode is chosen and validated exactly as in the reference (mb_svd_mode: "auto",
        "local-svd", "local-eigs", "dist-eigs", with its `require` messages).  Deliberate deviations, on every mode:
          * one Gramian G = A^T A on the device (split-K DMMA, summed in a fixed order) and one full eigendecomposition
            of G by parallel Jacobi; "dist-eigs" exists in the reference to keep n^2 doubles off the driver.  Device
            memory, not the 65535-column cap, bounds n: G, V and the eigensolver's four working copies take about
            48 * n^2 bytes besides A (about n = 40000 on an 80 GB H100; beyond that MarlinError MB_ERR_OOM).  Unlike
            ARPACK the result never has fewer than k values;
          * the Gramian's summation order differs from the reference's row-by-row dspr, so the results agree with it
            within rounding, not bitwise;
          * s = sqrt(|w|), the singular values of G as local-svd (dgesdd) returns them.
        Passing maxIter or tol selects the reference's full overload computeSVD(k, computeU, rCond, maxIter, tol, mode)
        (an omitted one takes the reference's default, max(300, 3k) or 1e-10), whose eigs modes run the restarted
        Lanczos solver (mb_eigs_*) for the k largest eigenvalues of G, chosen by mb_svd_plan: "local-eigs" forms G and
        applies it with mb_block_gemv; "dist-eigs" never forms G, its operator is mb_block_gram_matvec over the rows
        (any n up to 2^31 - 1, 8 n (2 ncv + 3) bytes of device memory besides A, ncv = min(2k, n)); "local-svd" is the
        Gramian and Jacobi path above.
        With several ranks every rank forms the Gramian of its rows (or, in dist-eigs, the product with its rows), zeros
        if it holds none; the partials are exchanged and summed in rank order on every rank, so all ranks hold the same
        bits and compute the same s and V.  The rows of U stay on the rank that holds the matching rows of this matrix."""
        import ctypes as C
        lib = nat.load()
        n = self.numCols()
        cm = C.c_int32()
        if maxIter is None and tol is None:
            nat.check(lib.mb_svd_mode(n, int(k), str(mode).encode(), C.byref(cm)))
            w, vblk = self._gramian().symmetricEigen()
            return self._svd_finish(w, vblk, int(k), computeU, rCond)
        maxIter = max(300, 3 * int(k)) if maxIter is None else int(maxIter)
        tol = 1e-10 if tol is None else float(tol)
        nat.check(lib.mb_svd_plan(n, int(k), str(mode).encode(), maxIter, tol, C.byref(cm)))
        if cm.value == nat.MB_SVD_LOCAL_LAPACK:
            w, vblk = self._gramian().symmetricEigen()
            return self._svd_finish(w, vblk, int(k), computeU, rCond)
        rt = Runtime.get()
        if cm.value == nat.MB_SVD_LOCAL_ARPACK:
            g = self._gramian()
            op = lambda x, y: nat.check(rt.lib.mb_block_gemv(rt.ctx, g.handle(), x, y, 0))
        else:
            op = self._gram_matvec_op(n)
        w, vblk, self.last_eigs_stats = symmetric_eigs(op, n, int(k), tol, maxIter)
        return self._svd_finish(w, vblk, int(k), computeU, rCond)

    def _gramian(self) -> SubMatrix:
        """G = A^T A over all ranks' rows, identical bits on every rank."""
        n = self.numCols()
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
        return g

    def _gram_matvec_op(self, n: int):
        """The dist-eigs operator y = sum over the ranks, in rank order, of A_r^T (A_r x)."""
        rt = Runtime.get()
        rank, ws = world()
        has_rows = self.data is not None and len(self.ids) > 0
        # every rank learns of a bad shard before any rank enters the exchanges
        problems = [(nat.MB_ERR_UNSUPPORTED, "computeSVD: fp64 rows only")] if has_rows and self.data.dtype != nat.MB_F64 else []
        problems = self._gather(problems)
        if problems:
            raise nat.MarlinArgumentError(*problems[0])
        if ws == 1:
            if not has_rows:
                raise nat.MarlinError(nat.MB_ERR_EMPTY, "empty collection")
            return lambda x, y: nat.check(rt.lib.mb_block_gram_matvec(rt.ctx, self.data.handle(), x, y, 0))
        dev = self.data.buf.device if self.data is not None else rt.device
        mine = SubMatrix.zeros(n, 1, nat.MB_F64, dev)
        sends = [(src, dst, ("gmv", src)) for src in range(ws) for dst in range(ws) if src != dst]

        def op(x, y):
            rt.sync_stream()
            if has_rows:
                nat.check(rt.lib.mb_block_gram_matvec(rt.ctx, self.data.handle(), x, mine.handle(), 0))
            got = comm.exchange(sends, {("gmv", rank): mine.buf}, lambda key: torch.empty(n, dtype=torch.float64, device=dev),
                                rank)
            parts = [mine if r == rank else SubMatrix(buf=got[("gmv", r)], rows=n, cols=1, ld=n) for r in range(ws)]
            total = parts[0]
            for p in parts[1:]:
                total = total.add(p)
            nat.check(rt.lib.mb_block_copy(rt.ctx, total.handle(), y))
        return op

    def _svd_finish(self, w: np.ndarray, vblk: SubMatrix, k: int, computeU: bool, rCond: float):
        """:1607-1652 from the eigenvalues w of G (in the solver's order) and their vectors, the columns of vblk."""
        lib = nat.load()
        n = vblk.rows
        dev = vblk.buf.device
        sigmas = np.sqrt(np.abs(w))
        sk = lib.mb_svd_rank(sigmas.ctypes.data_as(nat.c_dp), len(sigmas), k, float(rCond))
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

    # ------------------------------------------------------------------ logistic regression (:1005-1035)
    def lr(self, stepSize: float, iters: int) -> np.ndarray:
        """lr(stepSize, iters) :1005-1035 -> the weights (ndarray of numCols()).  Column 0 of every row is its label, the
        features are the row with column 0 replaced by the intercept 1; w starts at zeros, and iteration i = 1..iters sets
        w = w - delta * (stepSize / dataSize / sqrt(i)), delta the sum over all rows of features * gradientMul with
        gradientMul = 1 / (1 + exp(-1.0 * features.dot(w))) - label, and dataSize = numRows() (max row id + 1).

        On the device: each row's margin is sequential in column order with separate multiplies and adds (Breeze/F2J
        ddot bit for bit); the sum of the gradients runs in a fixed order, so the result is bitwise reproducible (the
        reference's reduce order follows task completion).  With one rank the whole loop runs on the GPU without host
        round trips (mb_lr_train).  With several ranks every rank computes the gradient sum of its rows each iteration
        (zeros if it holds none); the partials are exchanged and summed in rank order on every rank, so all ranks hold
        the same w bit for bit.  fp64 rows only."""
        n = self.numCols()
        data_size = self.numRows()
        rank, ws = world()
        has_rows = self.data is not None and len(self.ids) > 0
        iters = int(iters)
        w = np.zeros(n)
        if iters <= 0:
            return w
        # every rank learns of a bad shard before any rank enters the exchange below
        problems = []
        if has_rows and self.data.dtype != nat.MB_F64:
            problems.append((nat.MB_ERR_UNSUPPORTED, "lr: fp64 rows only"))
        elif has_rows and self.data.cols != n:
            # features.dot(weights) on rows of another length than the numCols() weights (Breeze's require)
            problems.append((nat.MB_ERR_DIM_MISMATCH, "requirement failed: Vectors must have the same length: rows of "
                             f"{self.data.cols} vs {n} weights"))
        problems = self._gather(problems)
        if problems:
            raise nat.MarlinArgumentError(*problems[0])
        rt = Runtime.get()
        if ws == 1:
            if not has_rows:
                raise nat.MarlinError(nat.MB_ERR_EMPTY, "empty collection")       # gradientRDD.reduce on no rows
            rt.sync_stream()
            nat.check(rt.lib.mb_lr_train(rt.ctx, self.data.handle(), data_size, float(stepSize), iters, w.ctypes.data_as(nat.c_dp)))
            return w
        import torch.distributed as dist
        # the partials are n doubles already on the host: NCCL moves them from the device, gloo from host memory
        dev = (self.data.buf.device if self.data is not None else rt.device) if dist.get_backend() == "nccl" else torch.device("cpu")
        for i in range(1, iters + 1):
            g = np.zeros(n)
            if has_rows:
                rt.sync_stream()
                nat.check(rt.lib.mb_lr_gradient(rt.ctx, self.data.handle(), w.ctypes.data_as(nat.c_dp), g.ctypes.data_as(nat.c_dp)))
            mine = torch.from_numpy(g).to(dev)
            sends = [(src, dst, ("lr", src)) for src in range(ws) for dst in range(ws) if src != dst]
            got = comm.exchange(sends, {("lr", rank): mine}, lambda key: torch.empty(n, dtype=torch.float64, device=dev), rank)
            parts = [g if r == rank else got[("lr", r)].cpu().numpy() for r in range(ws)]
            delta = parts[0].copy()
            for p in parts[1:]:
                delta = delta + p
            w = w - delta * (float(stepSize) / float(data_size) / math.sqrt(i))
        return w

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

    def _select_rows(self, positions, c0: int = 0, c1: Optional[int] = None) -> "DenseVecMatrix":
        """The local rows at `positions` (ascending local order), columns c0 until c1 (all by default), as a new packed
        row-major shard."""
        c1 = self.numCols() if c1 is None else c1
        nc = c1 - c0
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
            shard.slice(p, q + 1, 0, nc).assign(self.data.slice(positions[p], positions[q] + 1, c0, c1))
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

    # ------------------------------------------------------------------ norm (:975-999)
    def norm(self, mode: str) -> float:
        """norm(mode) :975-999 with mode "1" (the largest column sum of |a|), "inf" (the largest row sum of |a|) or "fro"
        (sqrt of the sum of a^2); any other mode, "2" included, is MarlinArgumentError "Do not support mode <mode>.".
        Deliberate deviations (DESIGN §3.14): the reference's "1" never sums (its per-row map is lazy and discarded) and
        its "inf" sums signed values; "fro" is a TODO there.

        One pass over each rank's shard on the device (mb_block_norm).  A NaN anywhere is the result (RDD.max() order).
        With several ranks the column sums of "1" and the accumulators of "fro" are exchanged and added in rank order on
        every rank; the row maxima of "inf" are combined by max, so "inf" is the same bits for any number of ranks.
        No rows on any rank is MarlinError MB_ERR_EMPTY "empty collection"."""
        import ctypes as C
        lib = nat.load()
        kind = C.c_int32()
        nat.check(lib.mb_norm_mode(str(mode).encode(), C.byref(kind)))
        kind = kind.value
        has_rows = self.data is not None and len(self.ids) > 0
        local = None
        if has_rows:
            rt = Runtime.get()
            rt.sync_stream()
            try:
                if kind == nat.MB_NORM_ONE:
                    col = SubMatrix.empty(self.data.cols, 1, nat.MB_F64, self.data.buf.device)
                    nat.check(rt.lib.mb_block_norm(rt.ctx, self.data.handle(), kind, col.handle(), None))
                    local = ("ok", col.toBreeze().reshape(-1))
                else:
                    out = np.zeros(3)
                    nat.check(rt.lib.mb_block_norm(rt.ctx, self.data.handle(), kind, None, out.ctypes.data_as(nat.c_dp)))
                    local = ("ok", out)
            except (nat.MarlinError, nat.MarlinArgumentError) as e:
                local = ("error", (e.code, getattr(e, "message", str(e))))
        # every rank learns of a failing shard before any rank raises; the error travels as (code, message)
        parts = self._gather([local] if local is not None else [])
        for status, value in parts:
            if status == "error":
                code, message = value
                if code in (nat.MB_ERR_INVALID_ARG, nat.MB_ERR_DIM_MISMATCH, nat.MB_ERR_UNSUPPORTED):
                    raise nat.MarlinArgumentError(code, message)
                raise nat.MarlinError(code, message)
        if not parts:
            raise nat.MarlinError(nat.MB_ERR_EMPTY, "empty collection")
        if kind == nat.MB_NORM_INF:
            vals = [float(v[0]) for _, v in parts]
            return math.nan if any(math.isnan(v) for v in vals) else max(vals)
        total = parts[0][1].copy()
        if kind == nat.MB_NORM_ONE:
            for _, v in parts[1:]:
                total = total + v
            return float(np.max(total))                        # np.max propagates NaN
        acc = np.ascontiguousarray(np.stack([v for _, v in parts]))
        res = C.c_double()
        nat.check(lib.mb_norm_fro(acc.ctypes.data_as(nat.c_dp), len(parts), C.byref(res)))
        return float(res.value)

    # ------------------------------------------------------------------ slicing (:928-964)
    def _window(self, r0: int, r1: int, c0: int, c1: int) -> "DenseVecMatrix":
        """Rows r0..r1 and columns c0..c1 (inclusive), row ids shifted by -r0; rows stay on their rank."""
        keep = [p for p, i in enumerate(self.ids) if r0 <= int(i) <= r1]
        nr, nc = r1 - r0 + 1, c1 - c0 + 1
        if not keep:
            return DenseVecMatrix(ids=np.zeros(0, dtype=np.int64), data=None, nRows=nr, nCols=nc)
        part = self._select_rows(keep, c0, c1 + 1)
        return DenseVecMatrix(ids=part.ids - r0, data=part.data, nRows=nr, nCols=nc)

    def sliceByRow(self, startRow: int, endRow: int) -> "DenseVecMatrix":
        """sliceByRow(startRow, endRow) :928-933 — rows startRow..endRow (inclusive) with ids shifted by -startRow.  The
        reference lets endRow == numRows() through (a phantom zero row); that is rejected here with its message."""
        if not (startRow >= 0 and endRow < self.numRows() and startRow <= endRow):
            raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, "start row or end row mismatch the matrix num of rows")
        return self._window(int(startRow), int(endRow), 0, self.numCols() - 1)

    def sliceByColumn(self, startCol: int, endCol: int) -> "DenseVecMatrix":
        """sliceByColumn(startCol, endCol) :941-946 — columns startCol..endCol (inclusive); endCol == numCols() (short rows
        in the reference) is rejected with its message."""
        if not (startCol >= 0 and endCol < self.numCols() and startCol <= endCol):
            raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, "start column or end column mismatch the matrix num of columns")
        return self._window(0, self.numRows() - 1, int(startCol), int(endCol))

    def getSubMatrix(self, startRow: int, endRow: int, startCol: int, endCol: int) -> "DenseVecMatrix":
        """getSubMatrix(startRow, endRow, startCol, endCol) :956-964 — inclusive bounds, row ids shifted by -startRow.  The
        reference's messages ("dismatch"), and also rejecting end == numRows() / numCols() and start > end."""
        if not (startRow >= 0 and endRow < self.numRows() and startRow <= endRow):
            raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, "start row or end row dismatch the matrix num of rows")
        if not (startCol >= 0 and endCol < self.numCols() and startCol <= endCol):
            raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, "start column or end column dismatch the matrix num of columns")
        return self._window(int(startRow), int(endRow), int(startCol), int(endCol))

    # ------------------------------------------------------------------ cBind (:238-252)
    def cBind(self, other):
        """cBind(other) :238-252 — rows.join(that.rows): a row id present on one side only is dropped; each remaining row
        is this row ++ that row, numRows() x (n1 + n2).  A BlockMatrix goes through toDenseVecMatrix() first."""
        from .block_matrix import BlockMatrix
        if isinstance(other, DistributedMatrix) and self.numRows() != other.numRows():
            raise nat.MarlinArgumentError(nat.MB_ERR_DIM_MISMATCH, f"Dimension mismatch:  {self.numRows()} vs {other.numRows()}")
        if isinstance(other, BlockMatrix):
            return self.cBind(other.toDenseVecMatrix())
        if not isinstance(other, DenseVecMatrix):
            raise nat.MarlinArgumentError(nat.MB_ERR_UNSUPPORTED, f"Do not support this type {type(other)} for cBind operation")
        n1, n2 = self.numCols(), other.numCols()
        theirs = set(int(i) for part in self._gather([other.ids.tolist()]) for i in part)
        keep = [p for p, i in enumerate(self.ids) if int(i) in theirs]
        me = self if len(keep) == len(self.ids) else self._select_rows(keep)
        that = other._aligned_to(me)                               # collective on every rank
        if me.data is None or not len(me.ids):
            return DenseVecMatrix(ids=me.ids, data=None, nRows=self.numRows(), nCols=n1 + n2)
        k = len(me.ids)
        buf = torch.empty(k * (n1 + n2), dtype=me.data.buf.dtype, device=me.data.buf.device)
        shard = SubMatrix(buf=buf, rows=k, cols=n1 + n2, ld=n1 + n2, is_transpose=True)
        shard.slice(0, k, 0, n1).assign(me.data)
        shard.slice(0, k, n1, n1 + n2).assign(that.data)
        return DenseVecMatrix(ids=me.ids, data=shard, nRows=self.numRows(), nCols=n1 + n2)

    # ------------------------------------------------------------------ MTUtils.repeatByRow / repeatByColumn (:446-491)
    def _repeat_columns(self, times: int) -> "DenseVecMatrix":
        """Every row becomes `times` copies of itself side by side (MTUtils.repeatByRow)."""
        n = self.numCols()
        if self.data is None or not len(self.ids):
            return DenseVecMatrix(ids=self.ids, data=None, nRows=self.numRows(), nCols=n * times)
        k = len(self.ids)
        buf = torch.empty(k * n * times, dtype=self.data.buf.dtype, device=self.data.buf.device)
        shard = SubMatrix(buf=buf, rows=k, cols=n * times, ld=max(1, n * times), is_transpose=True)
        for i in range(times):
            shard.slice(0, k, i * n, (i + 1) * n).assign(self.data)
        return DenseVecMatrix(ids=self.ids, data=shard, nRows=self.numRows(), nCols=n * times)

    def _repeat_rows(self, times: int) -> "DenseVecMatrix":
        """The matrix stacked `times` times: copy i of row id holds id + i * numRows() (MTUtils.repeatByColumn); every copy
        stays on the rank of its row."""
        m, n = self.numRows(), self.numCols()
        if self.data is None or not len(self.ids):
            return DenseVecMatrix(ids=np.zeros(0, dtype=np.int64), data=None, nRows=m * times, nCols=n)
        k = len(self.ids)
        buf = torch.empty(k * times * n, dtype=self.data.buf.dtype, device=self.data.buf.device)
        shard = SubMatrix(buf=buf, rows=k * times, cols=n, ld=max(1, n), is_transpose=True)
        for i in range(times):
            shard.slice(i * k, (i + 1) * k, 0, n).assign(self.data)
        ids = np.concatenate([self.ids + i * m for i in range(times)])
        return DenseVecMatrix(ids=ids, data=shard, nRows=m * times, nCols=n)

    # ------------------------------------------------------------------ transpose (:1420-1436)
    def transpose(self, numBlocks: Optional[int] = None):
        """toBlockMatrix(min(parallelism, rows/2), 1).transpose(); parallelism defaults to the number of GPUs
        (spark.default.parallelism), or 2 on one GPU to match the reference suite's local[2]."""
        rank, ws = world()
        par = numBlocks if numBlocks is not None else (ws if ws > 1 else 2)
        return self.toBlockMatrix(min(par, self.numRows() // 2), 1).transpose()

    # ------------------------------------------------------------------ rows -> blocks (:1084-1328)
    def toSparseVecMatrix(self):
        """:1333-1353 — the entries != 0.0 of every row (NaN kept, +-0.0 dropped) as a SparseVecMatrix, built on the
        device; its vectors have length numCols (the reference gives them length nnz)."""
        from .sparse_vec_matrix import SparseVecMatrix
        return SparseVecMatrix._from_dense(self)

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
        return BlockMatrix(res, mRows, mCols, by_row, by_col, sparse=False)

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
        """This rank's part file.  Device-resident rows are formatted by the device writer (mb_save_rows), which sends
        only text across PCIe; the host loop serves host-resident rows, which exist without a GPU only."""
        import os
        rank, ws = world()
        os.makedirs(path, exist_ok=True)
        part = os.path.join(path, f"part-{rank:05d}")
        has_rows = self.data is not None and len(self.ids) > 0
        on_device = self.data.buf.is_cuda if has_rows else Runtime.available()
        if on_device:
            import ctypes as C
            rt = Runtime.get()
            rt.sync_stream()
            ids = np.ascontiguousarray(self.ids, dtype=np.int64)
            nat.check(rt.lib.mb_save_rows(rt.ctx, self.data.handle() if has_rows else None,
                                          ids.ctypes.data_as(C.c_void_p) if has_rows else None, os.fsencode(part)))
            return
        from ..utils.mt_utils import _jdouble
        arr = self.data.toBreeze() if has_rows else np.zeros((0, 0))
        with open(part, "w") as fh:
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

"""CoordinateMatrix — the drop-in for edu.nju.pasalab.marlin.matrix.CoordinateMatrix (matrix/CoordinateMatrix.scala)
and its ALS (ml/ALSHelp.scala).

An RDD[((Long, Long), Float)] becomes, per rank, the entries this rank holds: int64 row ids, int64 column ids and float32
values.  ALS runs on the GPU: the links (ALSHelp's in/out-link blocks) are built by the library's host logic
(mb_als_links), the initial factors by mb_als_init_factors, and every half-step by one kernel that assembles and solves each
entity's normal equations (mb_als_update / mb_als_train).
"""
from __future__ import annotations

import ctypes as C
import re
import time
from typing import Tuple

import numpy as np
import torch

from .. import _native as nat
from .. import comm
from ..runtime import Runtime, world
from .dense_vec_matrix import DenseVecMatrix
from .sub_matrix import SubMatrix


def _ptr(a) -> C.c_void_p:
    return C.c_void_p(a.ctypes.data if isinstance(a, np.ndarray) else a.data_ptr())


def _raise_gathered(call) -> None:
    """Run `call` on every rank; if it failed on any rank, raise on every rank.  Of several "not positive definite"
    failures the one naming the lowest entity id is raised, as one rank would report it."""
    err = None
    try:
        call()
    except (nat.MarlinError, nat.MarlinArgumentError) as e:
        err = (isinstance(e, nat.MarlinArgumentError), e.code, nat.load().mb_last_error().decode("utf-8", "replace")
               if not isinstance(e, nat.MarlinArgumentError) else str(e))
    rank, ws = world()
    if ws > 1:
        import torch.distributed as dist
        everyone = [None] * ws
        dist.all_gather_object(everyone, err)
        errs = [x for x in everyone if x is not None]
    else:
        errs = [err] if err is not None else []
    if not errs:
        return

    def key(x):
        m = re.search(r"entity (\d+) are not positive definite", x[2])
        return (0, int(m.group(1))) if m else (1, 0)
    arg, code, msg = min(errs, key=key)
    if arg:
        raise nat.MarlinArgumentError(code, msg)
    raise nat.MarlinError(code, msg)


class _Links:
    """One side of the problem (users: ent = row ids; products: ent = column ids), laid out by mb_als_links."""

    def __init__(self, ent: np.ndarray, partner: np.ndarray, values: np.ndarray, num_blocks: int, num_partner_blocks: int):
        lib = nat.load()
        nnz = len(ent)
        ent, partner = np.ascontiguousarray(ent, np.int64), np.ascontiguousarray(partner, np.int64)
        values = np.ascontiguousarray(values, np.float32)
        cap = max(nnz, 1)
        self.ids = np.empty(cap, np.int64)
        self.block_offsets = np.empty(num_blocks + 1, np.int64)
        self.offsets = np.empty(cap + 1, np.int64)
        self.partners = np.empty(cap, np.int32)
        self.ratings = np.empty(cap, np.float32)
        self.work = np.empty(cap, np.int32)
        n = nat.c_i64()
        nat.check(lib.mb_als_links(nnz, _ptr(ent), _ptr(partner), _ptr(values), num_blocks, num_partner_blocks, _ptr(self.ids),
                                   _ptr(self.block_offsets), _ptr(self.offsets), _ptr(self.partners), _ptr(self.ratings),
                                   _ptr(self.work), C.byref(n)))
        self.n = n.value
        self.ids, self.offsets, self.work = self.ids[:self.n], self.offsets[:self.n + 1], self.work[:self.n]
        self.partners, self.ratings = self.partners[:nnz], self.ratings[:nnz]
        self.num_blocks = num_blocks

    def init_factors(self, seed: int, side: int, rank: int) -> np.ndarray:
        """ALSHelp.scala:60-74: block b's positions get the successive randomFactors of its own generator."""
        lib = nat.load()
        out = np.empty((self.n, rank))
        for b in range(self.num_blocks):
            lo, hi = int(self.block_offsets[b]), int(self.block_offsets[b + 1])
            if hi > lo:
                nat.check(lib.mb_als_init_factors(int(seed), side, b, rank, hi - lo, _ptr(out[lo:hi])))
        return out

    def to_device(self, device, work: np.ndarray = None):
        """The device arrays and the mb_als_side over them (the work list restricted to `work` if given)."""
        work = self.work if work is None else work
        keep = [torch.from_numpy(a).to(device) for a in (self.ids.astype(np.int32), self.offsets, self.partners,
                                                          self.ratings, np.ascontiguousarray(work, np.int32))]
        side = nat.AlsSide(len(work), *[t.data_ptr() for t in keep])
        return side, keep


class CoordinateMatrix:
    def __init__(self, entries=None, nRows: int = 0, nCols: int = 0):
        """entries: iterable of ((row, col), value) held by THIS rank (the reference's RDD content), or a tuple of arrays
        (rows, cols, values).  Values are Float (float32), as in the reference."""
        self._nRows, self._nCols = int(nRows), int(nCols)
        if isinstance(entries, tuple) and len(entries) == 3 and not np.isscalar(entries[0]):
            r, c, v = entries
        else:
            items = list(entries or [])
            r = [int(e[0][0]) for e in items]
            c = [int(e[0][1]) for e in items]
            v = [e[1] for e in items]
        self.rows = np.asarray(r, dtype=np.int64).reshape(-1)
        self.cols = np.asarray(c, dtype=np.int64).reshape(-1)
        self.values = np.asarray(v, dtype=np.float32).reshape(-1)
        if not (len(self.rows) == len(self.cols) == len(self.values)):
            raise nat.MarlinArgumentError(nat.MB_ERR_DIM_MISMATCH, "CoordinateMatrix: rows, cols and values differ in length")

    def _all_entries(self) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """Every rank's entries, concatenated in rank order (the same arrays on every rank)."""
        rank, ws = world()
        if ws == 1:
            return self.rows, self.cols, self.values
        import torch.distributed as dist
        parts = [None] * ws
        dist.all_gather_object(parts, (self.rows, self.cols, self.values))
        return tuple(np.concatenate([p[k] for p in parts]) for k in range(3))

    # ------------------------------------------------------------------ dims (:35-75)
    def _compute_size(self) -> None:
        rows, cols, _ = self._all_entries()
        if len(rows) == 0:
            raise nat.MarlinError(nat.MB_ERR_EMPTY, "empty collection")          # reduce on an empty RDD
        self._nRows = max(self._nRows, int(rows.max()) + 1)
        self._nCols = max(self._nCols, int(cols.max()) + 1)

    def numRows(self) -> int:
        if self._nRows <= 0:
            self._compute_size()
        return self._nRows

    def numCols(self) -> int:
        if self._nCols <= 0:
            self._compute_size()
        return self._nCols

    def toBreeze(self) -> np.ndarray:
        """:78-86 — a later entry for the same (row, col) wins, as in the reference's collect-and-assign."""
        m, n = self.numRows(), self.numCols()
        rows, cols, vals = self._all_entries()
        mat = np.zeros((m, n), order="F")
        mat[rows, cols] = vals.astype(np.float64)
        return mat

    def toDenseVecMatrix(self) -> DenseVecMatrix:
        """:51-64 — one row per row id that has entries (this rank takes a contiguous share of the sorted row ids), built
        on the device by mb_coo_to_dense_rows.  A repeated (row, col) fails as Vectors.sparse does."""
        n = self.numCols()
        if n > 2147483647:
            raise nat.MarlinError(nat.MB_ERR_UNSUPPORTED, f"Cannot convert to a row-oriented format because the number of "
                                  f"columns {n} is too large.")
        m = self.numRows()                                      # collective: before any rank can fail alone
        rows, cols, vals = self._all_entries()
        rank, ws = world()
        ids = np.unique(rows)
        lo, hi = (rank * len(ids)) // ws, ((rank + 1) * len(ids)) // ws
        mine = ids[lo:hi]
        sel = (rows >= mine[0]) & (rows <= mine[-1]) if len(mine) else np.zeros(len(rows), bool)
        rt = Runtime.get()
        data = None
        if len(mine):
            pos = np.ascontiguousarray(np.searchsorted(mine, rows[sel]), np.int32)
            c = np.ascontiguousarray(cols[sel], np.int32)
            v = np.ascontiguousarray(vals[sel], np.float32)
            buf = torch.empty(len(mine) * n, dtype=torch.float64, device=rt.device)
            data = SubMatrix(buf=buf, rows=len(mine), cols=n, ld=n, is_transpose=True)
            rt.sync_stream()

        def scatter():
            if data is not None:
                nat.check(rt.lib.mb_coo_to_dense_rows(rt.ctx, len(pos), _ptr(pos), _ptr(c), _ptr(v), data.handle()))
        _raise_gathered(scatter)                                # a duplicate on one rank fails every rank
        if data is None:
            return DenseVecMatrix([], m, n)
        return DenseVecMatrix(nRows=m, nCols=n, ids=mine, data=data)

    # ------------------------------------------------------------------ ALS (:88-98, ml/ALSHelp.scala:34-96)
    def ALS(self, rank: int, iterations: int, lambda_: float = 1.0, numUserBlock: int = 10, numProductBlock: int = 10,
            implicitPrefs: bool = False, alpha: float = 1.0, *, seed: int = None) -> Tuple[DenseVecMatrix, DenseVecMatrix]:
        """ALS(rank, iterations, lambda, numUserBlock, numProductBlock, implicitPrefs, alpha) -> (userFactors,
        productFactors), each a DenseVecMatrix whose row ids are the user (row) / product (column) ids and whose rows are
        the rank factors.  Users are hashed into numUserBlock blocks and products into numProductBlock blocks (-1: the
        number of ranks); the initial factors are the reference's (seed defaults to a time-based value, as
        System.nanoTime() there); each iteration updates the products from the users, then the users from the products.
        Deviations from the reference (DESIGN 3.10): the product of an entry is its column id; every user has its own
        normal equations; implicitPrefs uses the Gramian of the fixed side's factors as YtY; the solve is Cholesky; ids
        must lie in [0, 2^31 - 1].

        With several ranks, user and product block b are solved on rank b mod G; after each half-step the new rows are
        exchanged so every rank holds the whole fixed side.  Every entity's arithmetic is independent of its placement,
        so the factors are bit-identical to one rank's.  Each rank returns the rows of its own blocks."""
        rank_, iterations, lambda_, alpha = int(rank), int(iterations), float(lambda_), float(alpha)
        if seed is None:
            seed = time.monotonic_ns()
        me, ws = world()
        nub = ws if numUserBlock == -1 else int(numUserBlock)
        npb = ws if numProductBlock == -1 else int(numProductBlock)
        if rank_ < 1:
            raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, f"ALS: rank {rank_} must be at least 1")
        if rank_ > nat.MB_ALS_MAX_RANK:
            raise nat.MarlinArgumentError(nat.MB_ERR_UNSUPPORTED,
                                          f"ALS: rank {rank_} is above the kernel's cap of {nat.MB_ALS_MAX_RANK}")
        if not lambda_ >= 0.0:
            raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, f"ALS: lambda {lambda_} must be non-negative")
        if nub < 1 or npb < 1:
            raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, f"ALS: {nub} user and {npb} product blocks")
        rows, cols, vals = self._all_entries()                    # the same arrays, so the same decisions, on every rank
        if len(rows) == 0:
            raise nat.MarlinError(nat.MB_ERR_EMPTY, "empty collection")
        users = _Links(rows, cols, vals, nub, npb)
        products = _Links(cols, rows, vals, npb, nub)
        rt = Runtime.get()
        U = torch.from_numpy(users.init_factors(seed, 0, rank_)).to(rt.device)
        P = torch.from_numpy(products.init_factors(seed, 1, rank_)).to(rt.device)
        Ub = SubMatrix(buf=U.reshape(-1), rows=users.n, cols=rank_, ld=rank_, is_transpose=True)
        Pb = SubMatrix(buf=P.reshape(-1), rows=products.n, cols=rank_, ld=rank_, is_transpose=True)
        rt.sync_stream()
        if ws == 1:
            us, keep_u = users.to_device(rt.device)
            ps, keep_p = products.to_device(rt.device)
            nat.check(rt.lib.mb_als_train(rt.ctx, C.byref(us), C.byref(ps), iterations, lambda_, alpha, int(bool(implicitPrefs)),
                                          Ub.handle(), Pb.handle()))
            return (DenseVecMatrix(nRows=0, nCols=rank_, ids=users.ids.copy(), data=Ub),
                    DenseVecMatrix(nRows=0, nCols=rank_, ids=products.ids.copy(), data=Pb))
        own_u = self._own_work(users, me, ws)
        own_p = self._own_work(products, me, ws)
        us, keep_u = users.to_device(rt.device, own_u)
        ps, keep_p = products.to_device(rt.device, own_p)
        for _ in range(iterations):
            for side, links, Y, X, Xt in ((ps, products, Ub, Pb, P), (us, users, Pb, Ub, U)):
                # every rank learns of a failure on any rank before any rank enters the exchange
                _raise_gathered(lambda: nat.check(rt.lib.mb_als_update(rt.ctx, C.byref(side), Y.handle(), lambda_, alpha,
                                                                       int(bool(implicitPrefs)), None, X.handle())))
                self._share_rows(links, Xt, me, ws)
        return self._own_rows(users, U, me, ws, rank_), self._own_rows(products, P, me, ws, rank_)

    @staticmethod
    def _own_work(links: _Links, me: int, ws: int) -> np.ndarray:
        """The heaviest-first work list restricted to the blocks b with b mod G == this rank."""
        block = np.searchsorted(links.block_offsets, links.work, side="right") - 1
        return links.work[block % ws == me]

    @staticmethod
    def _share_rows(links: _Links, X: torch.Tensor, me: int, ws: int) -> None:
        """Every block's rows go from the rank that solved them to every other rank."""
        import torch.distributed as dist
        cpu = dist.get_backend() != "nccl"
        segs = {b: (int(links.block_offsets[b]), int(links.block_offsets[b + 1])) for b in range(links.num_blocks)}
        sends = [(b % ws, dst, b) for b, (lo, hi) in segs.items() if hi > lo for dst in range(ws) if dst != b % ws]
        local = {b: (X[lo:hi].cpu() if cpu else X[lo:hi].contiguous()) for b, (lo, hi) in segs.items() if b % ws == me and hi > lo}
        got = comm.exchange(sends, local, lambda b: torch.empty((segs[b][1] - segs[b][0], X.shape[1]), dtype=X.dtype,
                                                                device="cpu" if cpu else X.device), me)
        for b, t in got.items():
            X[segs[b][0]:segs[b][1]].copy_(t)

    @staticmethod
    def _own_rows(links: _Links, X: torch.Tensor, me: int, ws: int, rank_: int) -> DenseVecMatrix:
        pos = np.concatenate([np.arange(links.block_offsets[b], links.block_offsets[b + 1])
                              for b in range(links.num_blocks) if b % ws == me] or [np.zeros(0, np.int64)]).astype(np.int64)
        if not len(pos):
            return DenseVecMatrix([], 0, rank_)
        rows = X[torch.from_numpy(pos).to(X.device)].contiguous().reshape(-1)
        data = SubMatrix(buf=rows, rows=len(pos), cols=rank_, ld=rank_, is_transpose=True)
        return DenseVecMatrix(nRows=0, nCols=rank_, ids=links.ids[pos].copy(), data=data)

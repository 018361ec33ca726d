"""DistributedVector — the drop-in for edu.nju.pasalab.marlin.matrix.DistributedVector
(matrix/DistributedVector.scala): a long vector cut into `splitNum` pieces, each piece an (n x 1) block in HBM.

An RDD[(Int, DenseVector)] becomes `vectors`: the (id, piece) pairs THIS rank holds; piece `id` lives on rank
`id mod G` unless a placement callback says otherwise.  The arithmetic is the C ABI's vector kernels
(mb_block_gemv / mb_block_dot / mb_block_ger); pieces are small (8 bytes per element), so the exchange before a
matrix x vector product simply replicates them.
"""
from __future__ import annotations

import math
from typing import Callable, Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np
import torch

from .. import _native as nat
from .. import comm
from ..runtime import Runtime, world
from .block import BlockID
from .sub_matrix import SubMatrix


def _piece(v) -> SubMatrix:
    if isinstance(v, SubMatrix):
        if v.cols != 1:
            raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, "a vector piece is a block with one column")
        return v
    arr = np.asarray(v, dtype=np.float64).reshape(-1, 1)
    return SubMatrix(arr)


class DistributedVector:
    def __init__(self, vectors: Iterable[Tuple[int, object]], len: int = 0, splits: int = 0,      # noqa: A002
                 placement: Optional[Callable[[int], int]] = None):
        self.vectors: List[Tuple[int, SubMatrix]] = [(int(i), _piece(v)) for i, v in vectors]
        self._len, self._splits = int(len), int(splits)
        self._placement = placement
        self.columnMajor = True

    # ------------------------------------------------------------------ metadata (:24-43)
    def _gather(self, items: list) -> list:
        rank, ws = world()
        if ws == 1:
            return items
        import torch.distributed as dist
        out = [None] * ws
        dist.all_gather_object(out, items)
        return [x for part in out for x in part]

    def isColumnMajor(self) -> bool:
        return self.columnMajor

    def setColumnMajor(self, flag: bool) -> None:
        self.columnMajor = bool(flag)

    @property
    def splitNum(self) -> int:
        if self._splits <= 0:
            self._splits = len(self._gather([1 for _ in self.vectors]))
        return self._splits

    @property
    def length(self) -> int:
        if self._len <= 0:
            self._len = int(sum(self._gather([v.rows for _, v in self.vectors])))
        return self._len

    @property
    def getVectors(self):
        return self.vectors

    def owner(self, vec_id: int) -> int:
        rank, ws = world()
        if ws == 1:
            return 0
        return self._placement(vec_id) if self._placement is not None else vec_id % ws

    # ------------------------------------------------------------------ exchange
    def _replicated(self) -> Dict[int, SubMatrix]:
        """Every piece on every rank (the flatMap + join of BlockMatrix.scala:245-249 sends piece `id` to all m block
        rows; with one process per GPU that is one copy per rank)."""
        rank, ws = world()
        mine = {i: v for i, v in self.vectors}
        if ws == 1:
            return mine
        meta = sorted(self._gather([(i, v.rows, rank) for i, v in self.vectors]))
        lens = {i: n for i, n, _ in meta}
        sends = [(src, dst, i) for i, _, src in meta for dst in range(ws) if dst != src]
        local = {}
        for i, v in self.vectors:
            p = v if v.is_packed() else v.copy()
            local[i] = p.buf[: p.rows]
        dev = Runtime.get().device if Runtime.available() else torch.device("cpu")
        got = comm.exchange(sends, local, lambda i: torch.empty(lens[i], dtype=torch.float64, device=dev), rank)
        for i, buf in got.items():
            mine[i] = SubMatrix(buf=buf, rows=lens[i], cols=1, ld=max(1, lens[i]))
        return mine

    # ------------------------------------------------------------------ :45-73
    def substract(self, v: "DistributedVector") -> "DistributedVector":
        """(sic) element-wise difference of pieces with equal ids."""
        if self.length != v.length:
            raise nat.MarlinArgumentError(nat.MB_ERR_DIM_MISMATCH, f"unsupported vector length: {self.length} v.s {v.length}")
        theirs = v._replicated() if world()[1] > 1 else dict(v.vectors)
        res = [(i, p.subtract(theirs[i])) for i, p in self.vectors if i in theirs]
        return DistributedVector(res, v.length, self.splitNum, self._placement)

    def transpose(self) -> "DistributedVector":
        out = DistributedVector(self.vectors, self.length, self.splitNum, self._placement)
        out.setColumnMajor(False)
        return out

    def toBreeze(self) -> np.ndarray:
        """:65-73 — piece `id` starts at id * (length / pieces) (integer division, as written)."""
        pieces = self._gather([(i, v.toBreeze().reshape(-1)) for i, v in self.vectors])
        n = self.length
        out = np.zeros(n)
        offset = n // len(pieces)
        for i, arr in pieces:
            if i * offset + arr.shape[0] > n:
                raise IndexError("slice out of bounds")
            out[i * offset:i * offset + arr.shape[0]] = arr
        return out

    # ------------------------------------------------------------------ :84-107
    def toDisVector(self, splitStatusByRow: Sequence[Sequence[Tuple[int, Tuple[int, int], Tuple[int, int]]]],
                    splitNum: int) -> "DistributedVector":
        """Re-split: partition `p` (the p-th piece in id order) contributes elements [old0, old1] to elements
        [new0, new1] of new piece `vecId`.  Device-to-device slice copies."""
        n = self.length
        most = int(math.ceil(float(n) / float(splitNum)))
        rank, ws = world()
        src = self._replicated()
        order = sorted(src)
        new_ids = sorted({vec_id for st in splitStatusByRow for vec_id, _, _ in st})
        out: Dict[int, SubMatrix] = {}
        for vec_id in new_ids:
            if ws > 1 and vec_id % ws != rank:
                continue
            vlen = n - vec_id * most if (vec_id + 1) * most > n else most
            out[vec_id] = SubMatrix.zeros(vlen, 1)
        for pid, st in enumerate(splitStatusByRow):
            piece = src[order[pid]]
            for vec_id, (old0, old1), (new0, new1) in st:
                if vec_id in out:
                    out[vec_id].slice(new0, new1 + 1, 0, 1).assign(piece.slice(old0, old1 + 1, 0, 1))
        return DistributedVector(sorted(out.items()))

    # ------------------------------------------------------------------ :146-180
    def multiply(self, other: "DistributedVector", mode: str = "dist"):
        """column x row -> BlockMatrix of rank-1 blocks (Right in the reference's Either); row x column -> float (Left)."""
        from .block_matrix import BlockMatrix
        if self.length != other.length:
            raise nat.MarlinArgumentError(nat.MB_ERR_DIM_MISMATCH, "the length of these two vectors are not the same")
        if self.splitNum != other.splitNum:
            raise nat.MarlinArgumentError(nat.MB_ERR_UNSUPPORTED, "currently, only support two vectors with the same splits")
        rank, ws = world()
        if self.columnMajor and not other.columnMajor:
            s = self.splitNum
            mine, theirs = self._replicated(), other._replicated()
            rt = Runtime.get()
            blocks = []
            for i in sorted(mine):
                for j in range(s):
                    if j not in theirs or comm.elem_owner(i, j, s, ws) != rank:
                        continue
                    x, y = mine[i], theirs[j]
                    blk = SubMatrix.empty(x.rows, y.rows)
                    rt.sync_stream()
                    nat.check(rt.lib.mb_block_ger(rt.ctx, x.handle(), y.handle(), blk.handle()))
                    blocks.append((BlockID(i, j), blk))
            return BlockMatrix(blocks, self.length, self.length, s, s, sparse=False)
        if not self.columnMajor and other.columnMajor:
            m = mode.lower()
            if m == "dist":
                theirs = other._replicated() if ws > 1 else dict(other.vectors)
                parts = self._gather([(i, v.dot(theirs[i])) for i, v in self.vectors if i in theirs])
                if not parts:
                    raise nat.MarlinError(nat.MB_ERR_EMPTY, "empty collection")
                total = None
                for _, d in sorted(parts):                    # reduce(_ + _), ascending id
                    total = d if total is None else total + d
                return total
            if m == "local":
                a, b = SubMatrix(self.toBreeze().reshape(-1, 1)), SubMatrix(other.toBreeze().reshape(-1, 1))
                return a.dot(b)
            raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, "unrecognized mode")
        raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG,
                                      "the columnMajor status of the two distributed vectors are the same")

    # ------------------------------------------------------------------ companion (:184-190)
    @staticmethod
    def fromVector(sc, vector, numSplits: int) -> "DistributedVector":
        vector = np.asarray(vector, dtype=np.float64).reshape(-1)
        vlen = int(math.ceil(float(vector.shape[0]) / float(numSplits)))
        rank, ws = world()
        pieces = [(i, vector[i * vlen:min((i + 1) * vlen, vector.shape[0])]) for i in range(numSplits)
                  if ws == 1 or i % ws == rank]
        return DistributedVector(pieces, vector.shape[0], numSplits)

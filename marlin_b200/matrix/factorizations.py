"""Block LU / Cholesky / inverse of DenseVecMatrix on the GPU (SURVEY 8 f4; matrix/DenseVecMatrix.scala:283-764).

"breeze" mode (the reference collects the matrix and calls Breeze -> LAPACK) is one call into the recursive device
factorizations (`mb_block_lu / cholesky / inverse`, csrc/factor.cu).  "dist" mode is the reference's right-looking
block algorithm over a ceil(n / basesize)^2 grid; every block operation is a kernel of libmarlin_b200.so:

  LU        P_i A_ii = L_ii U_ii (pivoting inside the diagonal block only),  U_ic = L_ii^-1 (P_i A_ic),  L_ri = A_ri U_ii^-1,
            A_rc -= L_ri U_ic;  finally block row r of L is permuted by P_r                                   (:310-466)
  Cholesky  L_ii = chol(A_ii),  L_ri = A_ri L_ii^-T,  A_rc -= L_ri L_ci^T  (lower blocks only)                 (:497-556)
  inverse   elimination with inv(A_ii), then back substitution from the last block                            (:589-760)

The reference's permutation-matrix products (`(l \\ permutation) * block`, `permutation * blk`) are kept as products
with an uploaded 0/1 matrix (exact), its `block * brzInv(u)` / `blk * inv(l.t)` are triangular solves on transposed
views.

Sharding.  Block (r, c) lives on comm.elem_owner(r, c, nb, world) (MatrixElemOpPartitioner order) from the grid's
construction to the result, and every block operation runs on the rank that owns its output.  `plan_step` lists, for
one step of one algorithm, its phases: the operations each rank runs, then the blocks that move (one comm.exchange per
phase).  Every rank computes the same plan, so the exchanges match without negotiation.  The trailing update of a
step is one mb_block_schur_update call per rank (grouped DMMA launches), which gives each block the bits of today's
`multiply` + `subtract`; back substitution ships each product cur(r, c) * third(c, i) to the target's owner and adds
the products there in ascending c, the bits of the `multiply(..., accumulate=True)` chain.  So the result is the same
on any number of ranks.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

from .. import _native as nat
from .. import comm
from .block import BlockID
from .sub_matrix import SubMatrix

Blocks = Dict[Tuple[int, int], SubMatrix]
Key = tuple
Send = Tuple[int, int, Key]


def mode_is_dist(mode: str, n: int) -> bool:
    """:284-299 — "auto" switches to the distributed algorithm above 6000 rows."""
    if mode == "auto":
        return n > 6000
    if mode == "breeze":
        return False
    if mode == "dist":
        return True
    raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, f"Do not support mode {mode}.")


def grid(n: int, base: int):
    """:312-314 — numBlksByRow = ceil(n / basesize), block length = ceil(n / numBlksByRow)."""
    nb = int(math.ceil(n / float(base)))
    return nb, int(math.ceil(n / float(nb)))


# ---------------------------------------------------------------------------------------------------- the step plan
@dataclass(frozen=True)
class Op:
    rank: int
    name: str
    outs: Tuple[Key, ...]
    ins: Tuple[Key, ...]


@dataclass(frozen=True)
class Phase:
    ops: Tuple[Op, ...]          # run first, in order, each on its rank
    sends: Tuple[Send, ...]      # then one exchange of (src, dst, key)


KINDS = ("lu", "cholesky", "inverse", "inverse_back")


def steps(kind: str, nb: int) -> List[int]:
    """The step indices of an algorithm in execution order ("inverse_back" follows "inverse")."""
    return list(range(nb - 2, -1, -1)) if kind == "inverse_back" else list(range(nb))


def plan_step(kind: str, i: int, nb: int, world: int) -> List[Phase]:
    """Phases of step i.  Keys name blocks: ("A", r, c) the working block (r, c) (input, then factor); ("D", i) the
    packed LU factor of (i, i) with its pivots; ("I", i) inv(A_ii); ("T", r, i) = A_ri inv; ("S1", i, c) and
    ("S2", r, i) the scaled panels of the inverse; ("X", r, c) a block of the inverse; ("PT" | "PS" | "PF", i, ...)
    back-substitution products.  A key is held by the rank that produced it (or owns it), and by the ranks it is sent
    to until the end of the step."""
    if kind not in KINDS:
        raise ValueError(f"unknown factorization {kind}")
    o = lambda r, c: comm.elem_owner(r, c, nb, world)
    rest = range(i + 1, nb)
    sends: List[Send] = []

    def fan(src: int, key: Key, dsts) -> List[Send]:
        return [(src, d, key) for d in sorted(set(dsts)) if d != src]

    if kind == "lu":
        diag = (Op(o(i, i), "lu_diag", (("A", i, i), ("D", i)), (("A", i, i),)),)
        if i == nb - 1:
            return [Phase(diag, ())]
        d_sends = fan(o(i, i), ("D", i), [o(i, c) for c in rest] + [o(r, i) for r in rest])
        panel = tuple(Op(o(i, c), "lu_u", (("A", i, c),), (("D", i), ("A", i, c))) for c in rest) + \
            tuple(Op(o(r, i), "lu_l", (("A", r, i),), (("D", i), ("A", r, i))) for r in rest)
        for c in rest:
            sends += fan(o(i, c), ("A", i, c), [o(r, c) for r in rest])
        for r in rest:
            sends += fan(o(r, i), ("A", r, i), [o(r, c) for c in rest])
        update = tuple(Op(o(r, c), "schur", (("A", r, c),), (("A", r, c), ("A", r, i), ("A", i, c)))
                       for r in rest for c in rest)
        return [Phase(diag, tuple(d_sends)), Phase(panel, tuple(sends)), Phase(update, ())]

    if kind == "cholesky":
        diag = (Op(o(i, i), "chol_diag", (("A", i, i),), (("A", i, i),)),)
        if i == nb - 1:
            return [Phase(diag, ())]
        d_sends = fan(o(i, i), ("A", i, i), [o(r, i) for r in rest])
        panel = tuple(Op(o(r, i), "chol_l", (("A", r, i),), (("A", i, i), ("A", r, i))) for r in rest)
        for k in rest:
            sends += fan(o(k, i), ("A", k, i), [o(k, c) for c in range(i + 1, k + 1)] + [o(r, k) for r in range(k, nb)])
        update = tuple(Op(o(r, c), "schur_t", (("A", r, c),), (("A", r, c), ("A", r, i), ("A", c, i)))
                       for r in rest for c in range(i + 1, r + 1))
        return [Phase(diag, tuple(d_sends)), Phase(panel, tuple(sends)), Phase(update, ())]

    if kind == "inverse":
        if i == nb - 1:
            return [Phase((Op(o(i, i), "inv_last", (("X", i, i),), (("A", i, i),)),), ())]
        diag = (Op(o(i, i), "inv_diag", (("I", i),), (("A", i, i),)),)
        d_sends = fan(o(i, i), ("I", i), [o(i, c) for c in rest] + [o(r, i) for r in rest])
        panel = tuple(Op(o(r, i), "inv_third", (("T", r, i), ("S2", r, i)), (("I", i), ("A", r, i))) for r in rest) + \
            tuple(Op(o(i, c), "inv_second", (("S1", i, c),), (("I", i), ("A", i, c))) for c in rest)
        for r in rest:
            sends += fan(o(r, i), ("T", r, i), [o(r, c) for c in rest])
        for c in rest:
            sends += fan(o(i, c), ("A", i, c), [o(r, c) for r in rest])
        update = tuple(Op(o(r, c), "schur", (("A", r, c),), (("A", r, c), ("T", r, i), ("A", i, c)))
                       for r in rest for c in rest)
        return [Phase(diag, tuple(d_sends)), Phase(panel, tuple(sends)), Phase(update, ())]

    # inverse_back, step i < nb - 1: the blocks (r, i), (i, c), (i, i) of the inverse from the finished (r, c), r, c > i
    for c in rest:
        sends += fan(o(c, i), ("S2", c, i), [o(r, c) for r in rest])
    for r in rest:
        sends += fan(o(i, r), ("S1", i, r), [o(r, c) for c in rest] + [o(r, i)])
    products = tuple(Op(o(r, c), "mul", (("PT", i, r, c),), (("X", r, c), ("S2", c, i))) for r in rest for c in rest) + \
        tuple(Op(o(r, c), "mul", (("PS", i, r, c),), (("S1", i, r), ("X", r, c))) for r in rest for c in rest)
    p_sends = [(o(r, c), o(r, i), ("PT", i, r, c)) for r in rest for c in rest if o(r, c) != o(r, i)] + \
        [(o(r, c), o(i, c), ("PS", i, r, c)) for r in rest for c in rest if o(r, c) != o(i, c)]
    sums = tuple(Op(o(r, i), "sum", (("X", r, i),), tuple(("PT", i, r, c) for c in rest)) for r in rest) + \
        tuple(Op(o(i, c), "sum", (("X", i, c),), tuple(("PS", i, r, c) for r in rest)) for c in rest) + \
        tuple(Op(o(c, i), "mul", (("PF", i, c),), (("S1", i, c), ("X", c, i))) for c in rest)
    f_sends = [(o(c, i), o(i, i), ("PF", i, c)) for c in rest if o(c, i) != o(i, i)]
    first = (Op(o(i, i), "sum", (("X", i, i),), tuple(("PF", i, c) for c in rest) + (("I", i),)),)
    return [Phase((), tuple(sends)), Phase(products, tuple(p_sends)), Phase(sums, tuple(f_sends)), Phase(first, ())]


def key_shape(key: Key, size) -> Tuple[int, int]:
    """(rows, cols) of a block key; size(k) is the length of block row / column k."""
    name = key[0]
    if name in ("D", "I"):
        return size(key[1]), size(key[1])
    if name == "PT":
        return size(key[2]), size(key[1])
    if name == "PS":
        return size(key[1]), size(key[3])
    if name == "PF":
        return size(key[1]), size(key[1])
    return size(key[1]), size(key[2])


def _dead_after(kind: str, i: int, key: Key) -> bool:
    """Keys a rank may drop once step i has run (what it received is always dropped)."""
    name = key[0]
    if kind == "lu":
        return name == "D"
    if kind == "inverse":
        return name == "T" or (name == "A" and i in key[1:])
    if kind == "inverse_back":
        return name in ("PT", "PS", "PF") or key in (("I", i),) or (name == "S1" and key[1] == i) or \
            (name == "S2" and key[2] == i)
    return False


# ---------------------------------------------------------------------------------------------------- execution
def _perm_matrix(perm, device) -> SubMatrix:
    """permutation(j, p(j)) = 1 (:362-366): (P x)[j] = x[p[j]]."""
    n = len(perm)
    pm = np.zeros((n, n))
    pm[np.arange(n), np.asarray(perm)] = 1.0
    return SubMatrix(pm, device=device)


def _right_solve_upper(blk: SubMatrix, u: SubMatrix) -> SubMatrix:
    """X U = blk  <=>  U^T X^T = blk^T (U^T is lower triangular): `block * brzInv(u)` without forming the inverse."""
    return u.t.solveTriangular(blk.t, lower=True, unit=False).transpose()


def schur_update(entries: Sequence[Tuple[SubMatrix, SubMatrix, SubMatrix]]) -> None:
    """C -= A B in place for every (C, A, B): one mb_block_schur_update call."""
    from ..runtime import Runtime
    if not entries:
        return
    rt = Runtime.get(); rt.sync_stream()
    n = len(entries)
    arr = lambda j: (nat.c_blk * n)(*[e[j].handle() for e in entries])
    nat.check(rt.lib.mb_block_schur_update(rt.ctx, n, arr(0), arr(1), arr(2)))


def _flat(blk: SubMatrix) -> torch.Tensor:
    if not blk.is_packed():
        blk = blk.copy()
    return blk.buf[: blk.rows * blk.cols]


def _raise_same(problems: list, world: int) -> None:
    """Every rank raises the first failure of the phase (lowest rank) before anyone enters the next exchange."""
    if world > 1:
        import torch.distributed as dist
        out = [None] * world
        dist.all_gather_object(out, problems)
        problems = [p for part in out for p in part]
    if problems:
        code, msg = problems[0]
        cls = nat.MarlinArgumentError if code in (nat.MB_ERR_INVALID_ARG, nat.MB_ERR_DIM_MISMATCH,
                                                  nat.MB_ERR_UNSUPPORTED) else nat.MarlinError
        raise cls(code, msg)


def run(kind: str, store: Dict[Key, SubMatrix], nb: int, sub: int, n: int, rank: int, world: int, device,
        keep_unfactored_diagonal: bool = False, pivots: Dict[int, np.ndarray] = None) -> None:
    """Run every step of `kind` on this rank's blocks (store, updated in place)."""
    size = lambda k: n - sub * (nb - 1) if k == nb - 1 else sub
    for i in steps(kind, nb):
        got: Dict[Key, SubMatrix] = {}
        pm = None
        view = lambda k: got[k] if k in got else store[k]
        for phase in plan_step(kind, i, nb, world):
            mine = [op for op in phase.ops if op.rank == rank]
            problems = []
            try:
                schur = []
                for op in mine:
                    ins = [view(k) for k in op.ins]
                    if op.name in ("schur", "schur_t"):
                        schur.append((ins[0], ins[1], ins[2].t if op.name == "schur_t" else ins[2]))
                        continue
                    if op.name == "lu_diag":
                        packed, perm = ins[0].lu()
                        pivots[i] = perm
                        keep = keep_unfactored_diagonal and i < nb - 1
                        store[op.outs[0]] = ins[0] if keep else packed
                        store[op.outs[1]] = (packed, perm)
                        continue
                    if op.name in ("lu_u", "lu_l"):
                        packed, perm = ins[0]
                        if op.name == "lu_u":
                            if pm is None:
                                pm = _perm_matrix(perm, device)
                            store[op.outs[0]] = packed.solveTriangular(pm.multiply(ins[1]), lower=True, unit=True)
                        else:
                            store[op.outs[0]] = _right_solve_upper(ins[1], packed)
                        continue
                    outs = _OPS[op.name](*ins)
                    for k, v in zip(op.outs, outs if isinstance(outs, tuple) else (outs,)):
                        store[k] = v
                schur_update(schur)
            except (nat.MarlinError, nat.MarlinArgumentError) as e:
                if world == 1:
                    raise
                problems.append((e.code, str(e)))
            _raise_same(problems, world)
            if phase.sends and world > 1:
                local = {}
                for src, _, key in phase.sends:
                    if src == rank and key not in local:
                        v = view(key)
                        local[key] = torch.cat([_flat(v[0]), torch.as_tensor(v[1], dtype=torch.float64, device=device)]) \
                            if key[0] == "D" else _flat(v)

                def alloc(key):
                    r, c = key_shape(key, size)
                    return torch.empty(r * c + (r if key[0] == "D" else 0), dtype=torch.float64, device=device)

                for key, buf in comm.exchange(list(phase.sends), local, alloc, rank).items():
                    r, c = key_shape(key, size)
                    blk = SubMatrix(buf=buf, rows=r, cols=c, ld=max(1, r))
                    got[key] = (blk, buf[r * c:].cpu().numpy().astype(np.int64)) if key[0] == "D" else blk
        for k in [k for k in store if _dead_after(kind, i, k)]:
            del store[k]


def _sum(*blocks: SubMatrix) -> SubMatrix:
    acc = blocks[0]
    for b in blocks[1:]:
        acc.add_(b)
    return acc


_OPS = {
    "chol_diag": lambda a: a.cholesky(),           # reads the lower triangle (the reference first mirrors the upper one)
    "chol_l": lambda l, a: l.solveTriangular(a.t, lower=True, unit=False).transpose(),   # L L_ri^T = A_ri^T
    "inv_diag": lambda a: a.inverse(),
    "inv_last": lambda a: a.inverse(),
    "inv_third": lambda inv, a: (lambda t: (t, t.multiply(-1.0)))(a.multiply(inv)),
    "inv_second": lambda inv, a: inv.multiply(a).multiply(-1.0),
    "mul": lambda a, b: a.multiply(b),
    "sum": _sum,
}


def finish_lu(store: Dict[Key, SubMatrix], pivots: Dict[int, np.ndarray], nb: int, sub: int, n: int, rank: int,
              world: int, device):
    """The full pivot list on every rank, and block row r of L permuted by P_r on the blocks this rank holds."""
    items = [(i, [int(p) for p in perm]) for i, perm in pivots.items()]
    if world > 1:
        import torch.distributed as dist
        out = [None] * world
        dist.all_gather_object(out, items)
        items = [x for part in out for x in part]
    p_array = [0] * n
    for i, perm in items:
        for j, pj in enumerate(perm):
            p_array[i * sub + j] = i * sub + pj
    out: Blocks = {}
    for (name, r, c), blk in sorted((k, v) for k, v in store.items() if k[0] == "A"):
        if r > c:
            arr = p_array[sub * r: (n if r == nb - 1 else sub * r + sub)]
            blk = _perm_matrix([a - sub * r for a in arr], device).multiply(blk)
        out[(r, c)] = blk
    return out, p_array


def block_pairs(blocks: Blocks):
    return [(BlockID(r, c), b) for (r, c), b in sorted(blocks.items())]

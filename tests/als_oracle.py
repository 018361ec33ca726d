"""CoordinateMatrix.ALS (ml/ALSHelp.scala:34-403) restated step by step in numpy, for the tests.

- java.util.Random (nextInt, nextGaussian with its cached second value), scala.util.hashing.byteswap32 and randomFactor
  give the initial factors.
- The links follow makeOutLinkBlock / makeInLinkBlock and updateBlock's loops: positions by (block, id), a position's
  terms by (partner block, partner id, input order).
- assemble() sums every element of A_u and b_u in that order with separate IEEE roundings.  The sums are vectorised across
  entities and sequential across rating positions, so the per-element order is the reference's and the oracle stays fast.
- Solves are scipy's inv(A) @ b, as solveLeastSquares does.
- literal=True keeps the reference's defects: the product of an entry is its ROW id (:37), all users of a block share one
  XtX and one Xy (:304-307), and implicitPrefs fails on YtY.get of None (:79,81).
"""
from __future__ import annotations

import math
import struct
from dataclasses import dataclass

import numpy as np
import scipy.linalg

MASK48 = (1 << 48) - 1


def _i32(v: int) -> int:
    v &= 0xFFFFFFFF
    return v - (1 << 32) if v >= 1 << 31 else v


_LN2_HI, _LN2_LO = 6.93147180369123816490e-01, 1.90821492927058770002e-10
_LG = (6.666666666666735130e-01, 3.999999999940941908e-01, 2.857142874366239149e-01, 2.222219843214978396e-01,
       1.818357216161805012e-01, 1.531383769920937332e-01, 1.479819860511658591e-01)


def fdlibm_log(x: float) -> float:
    """java.lang.StrictMath.log (fdlibm e_log.c) for positive normal x, as nextGaussian calls it with 0 < x < 1.  The C
    library's log is not always the same in the last bit."""
    bits = struct.unpack("<q", struct.pack("<d", x))[0]
    hx, k = bits >> 32, 0
    assert 0x00100000 <= hx < 0x7FF00000
    k += (hx >> 20) - 1023
    hx &= 0x000FFFFF
    i = (hx + 0x95F64) & 0x100000
    x = struct.unpack("<d", struct.pack("<q", ((hx | (i ^ 0x3FF00000)) << 32) | (bits & 0xFFFFFFFF)))[0]
    k += i >> 20
    f = x - 1.0
    dk = float(k)
    if (0x000FFFFF & (2 + hx)) < 3:
        if f == 0.0:
            return 0.0 if k == 0 else dk * _LN2_HI + dk * _LN2_LO
        R = f * f * (0.5 - 0.33333333333333333 * f)
        return f - R if k == 0 else dk * _LN2_HI - ((R - dk * _LN2_LO) - f)
    s = f / (2.0 + f)
    z = s * s
    i = hx - 0x6147A
    w = z * z
    j = 0x6B851 - hx
    t1 = w * (_LG[1] + w * (_LG[3] + w * _LG[5]))
    t2 = z * (_LG[0] + w * (_LG[2] + w * (_LG[4] + w * _LG[6])))
    i |= j
    R = t2 + t1
    if i > 0:
        hfsq = 0.5 * f * f
        return f - (hfsq - s * (hfsq + R)) if k == 0 else dk * _LN2_HI - ((hfsq - (s * (hfsq + R) + dk * _LN2_LO)) - f)
    return f - s * (f - R) if k == 0 else dk * _LN2_HI - ((s * (f - R) - dk * _LN2_LO) - f)


class JavaRandom:
    """java.util.Random."""

    def __init__(self, seed: int):
        self.s = (seed ^ 0x5DEECE66D) & MASK48
        self.have_next = False
        self.next_next = 0.0

    def next(self, bits: int) -> int:
        self.s = (self.s * 0x5DEECE66D + 0xB) & MASK48
        return _i32(self.s >> (48 - bits))

    def next_int(self) -> int:
        return self.next(32)

    def next_double(self) -> float:
        return float((self.next(26) << 27) + self.next(27)) * 2.0 ** -53

    def next_gaussian(self) -> float:
        if self.have_next:
            self.have_next = False
            return self.next_next
        while True:
            v1 = 2 * self.next_double() - 1
            v2 = 2 * self.next_double() - 1
            s = v1 * v1 + v2 * v2
            if s < 1 and s != 0:
                break
        multiplier = math.sqrt(-2 * fdlibm_log(s) / s)    # StrictMath.sqrt / StrictMath.log
        self.next_next = v2 * multiplier
        self.have_next = True
        return v1 * multiplier


def byteswap32(v: int) -> int:
    """scala.util.hashing.byteswap32"""
    hc = (v * 0x9E3775CD) & 0xFFFFFFFF
    hc = int.from_bytes(hc.to_bytes(4, "little"), "big")
    return _i32(hc * 0x9E3775CD)


def random_factor(rank: int, rand: JavaRandom) -> np.ndarray:
    """ALSHelp.scala:170-179"""
    f = [abs(rand.next_gaussian()) for _ in range(rank)]
    s = 0.0
    for x in f:
        s = s + x * x
    norm = math.sqrt(s)
    return np.array([x / norm for x in f])


def seeds(seed: int):
    g = JavaRandom(seed)
    return g.next_int(), g.next_int()


@dataclass
class Links:
    ids: np.ndarray            # id of each position
    block_offsets: np.ndarray
    offsets: np.ndarray        # CSR over positions
    partners: np.ndarray       # partner position of each term
    ratings: np.ndarray        # float32
    work: np.ndarray           # heaviest first


def _positions(ids: np.ndarray, nb: int) -> np.ndarray:
    u = np.unique(ids)
    return u[np.lexsort((u, u % nb))]


def links(ent, partner, values, nb: int, npb: int) -> Links:
    ent, partner = np.asarray(ent, np.int64), np.asarray(partner, np.int64)
    for a in (ent, partner):
        if len(a) and (a.min() < 0 or a.max() > 2 ** 31 - 1):
            raise ValueError("id outside [0, 2147483647]")
    mine, theirs = _positions(ent, nb), _positions(partner, npb)
    # (block, id) order as one monotone key
    epos = np.searchsorted((mine % nb) * 2 ** 31 + mine, (ent % nb) * 2 ** 31 + ent)
    ppos = np.searchsorted((theirs % npb) * 2 ** 31 + theirs, (partner % npb) * 2 ** 31 + partner)
    order = np.lexsort((np.arange(len(ent)), ppos, epos))
    counts = np.bincount(epos, minlength=len(mine))
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    bo = np.concatenate([[0], np.cumsum(np.bincount(mine % nb, minlength=nb))]).astype(np.int64)
    return Links(mine, bo, offsets, ppos[order].astype(np.int32), np.asarray(values, np.float32)[order],
                 np.argsort(-counts, kind="stable").astype(np.int32))


def init_factors(L: Links, seed: int, side: int, rank: int) -> np.ndarray:
    """ALSHelp.scala:60-74"""
    s = seeds(seed)[side]
    out = np.empty((len(L.ids), rank))
    for b in range(len(L.block_offsets) - 1):
        rand = JavaRandom(byteswap32(s ^ b))
        for p in range(L.block_offsets[b], L.block_offsets[b + 1]):
            out[p] = random_factor(rank, rand)
    return out


def assemble(L: Links, Y: np.ndarray, lam: float, positions=None, implicit=False, alpha=1.0, yty=None):
    """(A, b) for the given positions (all by default): A packed lower, row-major (np.tril_indices order), regularisation
    and (implicit) YtY included, every element summed in the reference's order with separate roundings."""
    r = Y.shape[1]
    I, J = np.tril_indices(r)
    pos = np.arange(len(L.ids)) if positions is None else np.asarray(positions)
    cnt = L.offsets[pos + 1] - L.offsets[pos]
    order = np.argsort(-cnt, kind="stable")
    ps, cs = pos[order], cnt[order]
    A = np.zeros((len(ps), len(I)))
    b = np.zeros((len(ps), r))
    for q in range(int(cs.max()) if len(cs) else 0):
        k = int(np.count_nonzero(cs > q))
        idx = L.offsets[ps[:k]] + q
        y = Y[L.partners[idx]]
        rr = L.ratings[idx].astype(np.float64)
        t = y[:, I] * y[:, J]
        if not implicit:
            A[:k] = A[:k] + t
            b[:k] = b[:k] + rr[:, None] * y
        else:
            c = 1.0 + alpha * np.abs(rr)
            A[:k] = A[:k] + (c - 1.0)[:, None] * t
            m = rr > 0
            bk = b[:k]
            bk[m] = bk[m] + c[m][:, None] * y[m]
    diag = I == J
    A[:, diag] = A[:, diag] + (cs.astype(np.float64) * lam)[:, None]
    if implicit:
        A = A + yty[I, J][None, :]
    inv = np.empty_like(order)
    inv[order] = np.arange(len(order))
    return A[inv], b[inv]


def full(Ap: np.ndarray, r: int) -> np.ndarray:
    """fillFullMatrix"""
    I, J = np.tril_indices(r)
    M = np.zeros((r, r))
    M[I, J] = Ap
    M[J, I] = Ap
    return M


def gramian(Y: np.ndarray) -> np.ndarray:
    return Y.T @ Y


def half_step(L: Links, Y: np.ndarray, lam: float, implicit=False, alpha=1.0, yty=None, positions=None) -> np.ndarray:
    """updateBlock, corrected: every entity its own normal equations, solved as inv(A) @ b."""
    r = Y.shape[1]
    A, b = assemble(L, Y, lam, positions, implicit, alpha, yty)
    return np.stack([scipy.linalg.inv(full(A[k], r)) @ b[k] for k in range(len(A))]) if len(A) else np.zeros((0, r))


def _literal_half_step(L: Links, Y: np.ndarray, lam: float) -> np.ndarray:
    """updateBlock as written: per block one shared XtX / Xy summed over every term of every entity of the block in the
    loop order (partner block, partner id, group order); each entity adds only its own numRatings * lambda."""
    r = Y.shape[1]
    I, J = np.tril_indices(r)
    X = np.zeros((len(L.ids), r))
    for blk in range(len(L.block_offsets) - 1):
        lo, hi = L.block_offsets[blk], L.block_offsets[blk + 1]
        if hi == lo:
            continue
        q = np.arange(L.offsets[lo], L.offsets[hi])
        owner = np.repeat(np.arange(lo, hi), np.diff(L.offsets[lo:hi + 1]))
        # partners ascending; within one partner the CSR's order (owner ascending) stands in for the group's input order,
        # which only the last bits of the shared sums depend on
        q = q[np.argsort(L.partners[q], kind="stable")]
        Ap = np.zeros(len(I))
        b = np.zeros(r)
        for t in q:
            y = Y[L.partners[t]]
            Ap = Ap + y[I] * y[J]
            b = b + float(L.ratings[t]) * y
        for p in range(lo, hi):
            M = full(Ap, r)
            M[np.diag_indices(r)] = M[np.diag_indices(r)] + float(L.offsets[p + 1] - L.offsets[p]) * lam
            X[p] = scipy.linalg.inv(M) @ b
    return X


def als(rows, cols, values, rank: int, iterations: int, lam: float = 1.0, nub: int = 10, npb: int = 10,
        implicit: bool = False, alpha: float = 1.0, seed: int = 0, literal: bool = False):
    """ALSRun -> (user ids, U, product ids, P)."""
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    if literal:
        cols = rows                                            # Rating(r._1._1.toInt, r._1._1.toInt, r._2)
    users = links(rows, cols, values, nub, npb)
    products = links(cols, rows, values, npb, nub)
    U = init_factors(users, seed, 0, rank)
    P = init_factors(products, seed, 1, rank)
    for _ in range(iterations):
        if literal:
            if implicit:
                raise LookupError("None.get")                  # YtY = None, then YtY.get.value
            P = _literal_half_step(products, U, lam)
            U = _literal_half_step(users, P, lam)
        else:
            P = half_step(products, U, lam, implicit, alpha, gramian(U) if implicit else None)
            U = half_step(users, P, lam, implicit, alpha, gramian(P) if implicit else None)
    return users.ids, U, products.ids, P


def dense_masked_als(R: np.ndarray, mask: np.ndarray, U: np.ndarray, P: np.ndarray, lam: float, iterations: int):
    """An independent explicit ALS on a dense rating matrix with a 0/1 mask (no duplicates): the normal equations from
    matrix products, solved by np.linalg.solve."""
    r = U.shape[1]
    for _ in range(iterations):
        for j in range(R.shape[1]):
            S = mask[:, j].astype(bool)
            Y = U[S]
            P[j] = np.linalg.solve(Y.T @ Y + lam * S.sum() * np.eye(r), Y.T @ R[S, j])
        for i in range(R.shape[0]):
            S = mask[i].astype(bool)
            Y = P[S]
            U[i] = np.linalg.solve(Y.T @ Y + lam * S.sum() * np.eye(r), Y.T @ R[i, S])
    return U, P

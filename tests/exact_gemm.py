"""Integer-valued fp64 operands whose products are exact in every summation order, and the report of a mismatch.

If every operand is an integer and every partial sum of alpha * sum_k a_ik b_kj + beta * c_ij has magnitude at most
2^53, fp64 represents every intermediate exactly: any k order, any split of K, any DMMA shape and any host BLAS give the
same number.  A kernel can then be compared with `==` against plain `A @ B` in numpy, whatever order it sums in.

The operands are chosen so that the worst case |alpha| * K * max|a| * max|b| + |beta| * max|c| lies in [2^52, 2^53]:
the results use the whole 53-bit significand, so an accumulation narrower than fp64 or a dropped term changes them.
With a fractional alpha = 2^-p (or any dyadic alpha) the results are multiples of 2^-p and the bound counts in that
unit: alpha * 2^p and beta * 2^p are integers and the worst case, times 2^p, must lie in [2^52, 2^53].
"""
from __future__ import annotations

import math

import numpy as np

TWO52, TWO53 = 2 ** 52, 2 ** 53
TILE = 128


def unit_exponent(alpha: float, beta: float = 0.0) -> int:
    """The least p >= 0 with alpha * 2^p and beta * 2^p integers (results are multiples of 2^-p)."""
    for p in range(64):
        if float(alpha * 2.0 ** p).is_integer() and float(beta * 2.0 ** p).is_integer():
            return p
    raise ValueError(f"alpha = {alpha!r}, beta = {beta!r} are not dyadic")


def _max_int(x) -> int:
    """max |x| of an integer-valued array as a Python int (0 for an empty one); refuses non-integers."""
    x = np.asarray(x, dtype=np.float64)
    if x.size == 0:
        return 0
    if not np.all(np.isfinite(x)) or not np.array_equal(x, np.trunc(x)):
        raise ValueError("operands must be finite and integer-valued")
    return int(np.abs(x).max())


def worst_case(K: int, amax: int, bmax: int, alpha: float = 1.0, beta: float = 0.0, cmax: int = 0) -> int:
    """|alpha| K amax bmax + |beta| cmax in units of 2^-p, computed with Python ints: a bound on every partial sum."""
    p = unit_exponent(alpha, beta)
    ia, ib = abs(int(alpha * 2 ** p)), abs(int(beta * 2 ** p))
    return ia * int(K) * int(amax) * int(bmax) + ib * int(cmax)


def check_bound(A, B, alpha: float = 1.0, beta: float = 0.0, C0=None) -> int:
    """Assert that op = alpha A B + beta C0 is exact in fp64 in any order: integer operands and worst case <= 2^53 (in
    units of 2^-p).  Returns the worst case."""
    A, B = np.asarray(A), np.asarray(B)
    if A.ndim != 2 or B.ndim != 2 or A.shape[1] != B.shape[0]:
        raise ValueError(f"shapes {A.shape} x {B.shape}")
    cmax = _max_int(C0) if (C0 is not None and beta != 0.0) else 0
    w = worst_case(A.shape[1], _max_int(A), _max_int(B), alpha, beta, cmax)
    assert w <= TWO53, f"worst case {w} = 2^{math.log2(w):.4f} exceeds 2^53: the product is not exact in every order"
    return w


def magnitudes(K: int, alpha: float = 1.0, beta: float = 0.0, square: bool = False):
    """(amax, bmax, cmax) with worst_case(K, amax, bmax, alpha, beta, cmax) in [2^52, 2^53].  The addend takes at most
    2^51 units when beta != 0; square: amax == bmax (a Gramian, where both factors are the same matrix)."""
    if K < 1:
        raise ValueError("K >= 1")
    p = unit_exponent(alpha, beta)
    ia, ib = abs(int(alpha * 2 ** p)), abs(int(beta * 2 ** p))
    cmax = (2 ** 51) // ib if ib else 0
    q = (TWO53 - ib * cmax) // (ia * K)          # amax * bmax may not exceed this
    amax = math.isqrt(q)
    bmax = amax if square else q // amax
    if amax < 1:
        raise ValueError(f"K = {K} is too long for an exact product")
    return amax, bmax, cmax


def operands(rng, m: int, k: int, n: int, alpha: float = 1.0, beta: float = 0.0):
    """Integer A (m x k), B (k x n) and, for beta != 0, C0 (m x n) at the magnitudes of `magnitudes`: uniform with
    mixed signs (so sums cancel), and row 0 of A / column 0 of B of full magnitude with matching signs, so that
    result (0, 0) is exactly the worst case and uses the top bit of the bound."""
    amax, bmax, cmax = magnitudes(k, alpha, beta)
    A = rng.integers(-amax, amax + 1, size=(m, k)).astype(np.float64)
    B = rng.integers(-bmax, bmax + 1, size=(k, n)).astype(np.float64)
    s = rng.choice([-1.0, 1.0], size=k)
    A[0, :] = amax * s
    B[:, 0] = bmax * s
    C0 = None
    if beta != 0.0:
        C0 = rng.integers(-cmax, cmax + 1, size=(m, n)).astype(np.float64)
        C0[0, 0] = cmax * np.sign(alpha * beta)
    return A, B, C0


def gram_operand(rng, m: int, n: int):
    """Integer A (m x n) for G = A^T A: column 0 of full magnitude, so G(0, 0) is the worst case m * amax^2."""
    amax = magnitudes(m, square=True)[0]
    A = rng.integers(-amax, amax + 1, size=(m, n)).astype(np.float64)
    A[:, 0] = amax * rng.choice([-1.0, 1.0], size=m)
    return A


def reference(A, B, alpha: float = 1.0, beta: float = 0.0, C0=None):
    """alpha A B + beta C0 in numpy float64: exact (any BLAS order) once check_bound holds."""
    check_bound(A, B, alpha, beta, C0)
    out = alpha * (A @ B)
    if beta != 0.0:
        out = out + beta * C0
    return out


def report(got, want, tile: int = TILE) -> str:
    """Where and how got differs from want: the count, the bounding box of the wrong (i, j) and the tile ids it covers,
    and how many wrong values are NaN (never written) or finite but off (wrong terms)."""
    got, want = np.asarray(got), np.asarray(want)
    if got.shape != want.shape:
        return f"shape {got.shape} != {want.shape}"
    bad = ~((got == want) | (np.isnan(got) & np.isnan(want)))
    idx = np.argwhere(bad)
    if idx.size == 0:
        return "no difference"
    (i0, j0), (i1, j1) = idx.min(axis=0), idx.max(axis=0)
    g, w = got[bad], want[bad]
    nan = int(np.isnan(g).sum())
    fin = np.isfinite(g)
    off = np.abs(g[fin] - w[fin])
    first = tuple(int(v) for v in idx[0])
    return (f"{int(bad.sum())} of {bad.size} elements wrong in rows {i0}..{i1}, columns {j0}..{j1} "
            f"(tiles {i0 // tile}..{i1 // tile} x {j0 // tile}..{j1 // tile} of {tile}x{tile}); "
            f"{nan} NaN (never written), {int(fin.sum())} finite and off"
            + (f" by {off.min():.6g}..{off.max():.6g}, {int(np.sum(off == np.trunc(off)))} by an integer" if fin.any() else "")
            + f"; first at {first}: got {got[first]!r}, want {want[first]!r}")


def assert_exact(got, want, what="") -> None:
    """np.array_equal as numbers (NaN != NaN, -0.0 == +0.0), with `report` as the message."""
    if not np.array_equal(got, want):
        raise AssertionError(f"{what}: {report(got, want)}")

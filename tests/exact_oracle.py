"""Exact and high-precision references for the fp64 factorizations and the eigensolver.

* `getf2_exact`: LAPACK dgetf2 (partial-pivoting LU, first maximal |a| wins) in `fractions.Fraction` arithmetic, with
  dgetf2's choice between scaling by the reciprocal of the pivot (|pivot| >= sfmin = DBL_MIN) and dividing by it.  It also
  reports whether every value it formed — each reciprocal it multiplies by, each multiplier, each updated entry — is an
  fp64 number.  When that holds, an fp64 implementation that makes the same pivot choices computes every one of those
  values without rounding, in any summation order, so its factors must equal these bit for bit.
* `cholesky_int`: the Cholesky factor of an integer matrix that is L L^T for an integer L, in integer arithmetic.
* `eigvalsh_mp`: eigenvalues of a symmetric fp64 matrix by mpmath, to a chosen number of significant digits relative to
  each eigenvalue (the working precision is raised by the matrix's exponent range, since mpmath's solver is accurate
  relative to the norm of the matrix, not to each eigenvalue).
"""
from __future__ import annotations

import math
import sys
from fractions import Fraction

import numpy as np

SFMIN = sys.float_info.min          # dlamch('S') for IEEE double: 2^-1022


def representable(q: Fraction) -> bool:
    """True when q is exactly an fp64 number (finite)."""
    try:
        f = float(q)
    except OverflowError:
        return False
    return math.isfinite(f) and Fraction(f) == q


def getf2_exact(A):
    """dgetf2 on an m x n fp64 matrix in exact arithmetic.

    Returns (lu, ipiv, exact): lu packed like dgetrf (unit-lower L below the diagonal, U on and above it), the exact
    values rounded once to fp64, ipiv the 0-based interchanges (row c was swapped with row ipiv[c]), and `exact`.  `exact` is True when
      * every reciprocal used is an fp64 number, and
      * every multiplier is an fp64 number, and
      * for every entry (r, j), its input and every product l_rc u_cj subtracted from it are multiples of one 2^-q with
        (|a_rj| + sum_c |l_rc u_cj|) * 2^q < 2^53.
    Then every partial sum of every entry's update, taken in any order or grouping (a blocked, recursive or tensor-core
    update), is an fp64 number, and an implementation that makes the same pivot choices returns `lu` bit for bit."""
    A = np.asarray(A, dtype=np.float64)
    m, n = A.shape
    a = [[Fraction(float(v)) for v in row] for row in A]
    bound = [[abs(v) for v in row] for row in a]      # |a_rj| + sum |l u| so far, permuted along with the rows
    den = [[v.denominator for v in row] for row in a]  # the largest denominator among them
    exact = True
    ipiv = []
    for c in range(min(m, n)):
        p = c
        for r in range(c + 1, m):                      # idamax: the first row of the largest |a|
            if abs(a[r][c]) > abs(a[p][c]):
                p = r
        ipiv.append(p)
        if p != c:
            a[c], a[p] = a[p], a[c]
            bound[c], bound[p] = bound[p], bound[c]
            den[c], den[p] = den[p], den[c]
        pv = a[c][c]
        if pv == 0:
            continue                                   # singular column: dgetf2 records INFO and goes on
        recip = abs(pv) >= SFMIN
        rinv = 1 / pv
        if recip and any(a[r][c] for r in range(c + 1, m)):
            exact &= representable(rinv)             # only matters when it scales a nonzero entry
        for r in range(c + 1, m):
            lval = a[r][c] * rinv if recip else a[r][c] / pv
            a[r][c] = lval
            exact &= representable(lval)
            if lval:
                row_r, row_c, b_r, d_r = a[r], a[c], bound[r], den[r]
                for j in range(c + 1, n):
                    prod = lval * row_c[j]
                    row_r[j] -= prod
                    b_r[j] += abs(prod)
                    d_r[j] = max(d_r[j], prod.denominator)
    for r in range(m):
        for j in range(n):
            d = den[r][j]
            exact &= (d & (d - 1)) == 0 and bound[r][j] * d < 2 ** 53      # dyadic, and 53 bits hold every partial sum
    lu = np.array([[float(v) for v in row] for row in a])
    return lu, np.array(ipiv, dtype=np.int64), exact


def perm_from_ipiv(ipiv, m):
    """The reference's permutation array (row i of L U is row perm[i] of A) from dgetrf-style interchanges."""
    perm = np.arange(m)
    for i, p in enumerate(ipiv):
        perm[i], perm[p] = perm[p], perm[i]
    return perm


def cholesky_int(A):
    """L with A = L L^T, L integer lower triangular with a positive diagonal, from an integer-valued A; raises
    ValueError when A has no such factor (a pivot that is not a perfect square, or a division with a remainder)."""
    A = np.asarray(A)
    n = A.shape[0]
    a = [[int(v) for v in row] for row in A]
    L = [[0] * n for _ in range(n)]
    for j in range(n):
        d = a[j][j] - sum(L[j][k] * L[j][k] for k in range(j))
        r = math.isqrt(d) if d > 0 else -1
        if r <= 0 or r * r != d:
            raise ValueError(f"pivot {j} is {d}, not a positive perfect square")
        L[j][j] = r
        for i in range(j + 1, n):
            s = a[i][j] - sum(L[i][k] * L[j][k] for k in range(j))
            q, rem = divmod(s, r)
            if rem:
                raise ValueError(f"L[{i}][{j}] = {s}/{r} is not an integer")
            L[i][j] = q
    return L


def eigvalsh_mp(G, digits=40):
    """Eigenvalues of the symmetric fp64 matrix G (ascending, as Python floats), each to about `digits` significant
    digits: mpmath's symmetric solver at a working precision of `digits` plus the decimal exponent range of G's
    nonzero entries (its error is relative to ||G||, which must be that far below the smallest eigenvalue's rounding)."""
    import mpmath
    G = np.asarray(G, dtype=np.float64)
    nz = np.abs(G[G != 0])
    spread = 0 if nz.size == 0 else math.ceil(math.log10(nz.max()) - math.log10(nz.min()))
    with mpmath.workdps(digits + 2 * spread + 10):
        M = mpmath.matrix(G.tolist())
        E = mpmath.eigsy(M, eigvals_only=True)
        return sorted(float(E[i]) for i in range(G.shape[0]))

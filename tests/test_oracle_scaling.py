"""The premises of tests/test_gpu_late_kernel_edges.py, checked on the CPU: the host references of those kernels obey the
same exact power-of-two scaling on the same kinds of cases.  If a GPU scaling test fails, the invariant it rests on holds
here, so the kernel is at fault."""
import math

import numpy as np
import pytest
import scipy.linalg

from tests import als_oracle as ao
from tests import dms_api_oracle as do
from tests import pagerank_oracle as po
from tests import sparse_oracle as so
from tests import spvec_oracle as sv


def p2(k):
    return math.ldexp(1.0, int(k))


def identical(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.int64), b.view(np.int64))


def away_from_zero(rng, shape, lo=0.5):
    return np.where(rng.random(shape) < 0.5, -1.0, 1.0) * (lo + (1 - lo) * rng.random(shape))


def _als_case(rank, seed, implicit):
    rng = np.random.default_rng(seed)
    rows = np.concatenate([rng.integers(0, 40, 2400), np.full(300, 3)])
    cols = rng.integers(0, 60, len(rows))
    vals = rng.uniform(-3.0 if implicit else 0.5, 5.0, len(rows)).astype(np.float32)
    L = ao.links(rows, cols, vals, 3, 4)
    return L, away_from_zero(rng, (len(np.unique(cols)), rank))


@pytest.mark.parametrize("implicit", [False, True])
@pytest.mark.parametrize("rank", [10, 11, 32, 33, 50, 51])
def test_als_assembly_and_solve_scale_exactly(rank, implicit):
    """Y -> 2^k Y, lambda -> 4^k lambda (YtY -> 4^k YtY): A -> 4^k A, b -> 2^k b, and both the oracle's inv(A) b and a
    Cholesky solve give x -> 2^-k x."""
    L, Y = _als_case(rank, rank, implicit)
    lam, alpha = 0.05, 0.37
    yty = ao.gramian(Y) if implicit else None
    A0, b0 = ao.assemble(L, Y, lam, implicit=implicit, alpha=alpha, yty=yty)
    X0 = ao.half_step(L, Y, lam, implicit, alpha, yty)
    C0 = [scipy.linalg.cho_solve(scipy.linalg.cho_factor(ao.full(A0[p], rank), lower=True), b0[p]) for p in range(0, len(A0), 9)]
    for k in (1, -1, 37, -37, 250, -250):
        s = None if yty is None else yty * p2(2 * k)
        A, b = ao.assemble(L, Y * p2(k), lam * p2(2 * k), implicit=implicit, alpha=alpha, yty=s)
        assert identical(A, np.ldexp(A0, 2 * k)) and identical(b, np.ldexp(b0, k)), k
        assert identical(ao.half_step(L, Y * p2(k), lam * p2(2 * k), implicit, alpha, s), np.ldexp(X0, -k)), k
        for c0, p in zip(C0, range(0, len(A0), 9)):
            x = scipy.linalg.cho_solve(scipy.linalg.cho_factor(ao.full(A[p], rank), lower=True), b[p])
            assert identical(x, np.ldexp(c0, -k)), (k, p)


@pytest.mark.parametrize("kind", ["ds", "sd", "ss"])
def test_sparse_loops_scale_exactly(kind):
    rng = np.random.default_rng(len(kind) + ord(kind[0]))
    m, k, n = 1100, 60, 20
    csc = lambda r, c: so.csc_from_dense_pattern(away_from_zero(rng, (r, c)), rng.random((r, c)) < 0.1)
    scale = lambda X, e: X * p2(e) if isinstance(X, np.ndarray) else X[:4] + (X[4] * p2(e),)
    if kind == "ds":
        left, right, f = away_from_zero(rng, (m, k)), csc(k, n), so.mult_dense_sparse
    elif kind == "sd":
        left, right, f = csc(m, k), away_from_zero(rng, (k, n)), so.mult_sparse_dense
    else:
        left, right, f = csc(m, k), csc(k, n), so.spgemm
    C0 = away_from_zero(rng, (m, n))
    base = f(left, right)
    for a, b in [(1, 0), (0, -1), (37, -37), (500, -1), (-500, 1), (450, 450), (-450, -450)]:
        got = f(scale(left, a), scale(right, b))
        assert identical(got, np.ldexp(base, a + b)), (a, b)
        assert identical(C0 * p2(a + b) + got, np.ldexp(C0 + base, a + b)), (a, b)


def test_spvec_float32_products_scale_exactly_inside_float_range():
    """The fixed-order float32 sums: (2^a A)(2^b B) with |a + b| <= 100, |a|, |b| <= 60 and values of magnitude
    [0.5, 1) is 2^(a+b) times the unscaled result, bit for bit; past float's range it is not."""
    rng = np.random.default_rng(7)
    K, n = 300, 400
    B = [(k, np.sort(rng.choice(n, 40, replace=False)), away_from_zero(rng, 40)) for k in range(K)]
    A = [(i, np.sort(rng.choice(K, c, replace=False)), away_from_zero(rng, c)) for i, c in enumerate([1, 6, 7, 100, 103, 250])]
    scale = lambda rows, e: [(i, ix, v * p2(e)) for i, ix, v in rows]
    r0, c0, v0 = sv.multiply_sparse(A, B)
    for a, b in [(1, 0), (0, -1), (37, -37), (60, 40), (-60, -40), (60, -60)]:
        r, c, v = sv.multiply_sparse(scale(A, a), scale(B, b))
        assert np.array_equal(r, r0) and np.array_equal(c, c0)
        assert np.array_equal(v.view(np.uint32), np.ldexp(v0, a + b).astype(np.float32).view(np.uint32)), (a, b)
    _, _, v = sv.multiply_sparse(scale(A, 64), scale(B, 63))
    assert np.isinf(v).any()


@pytest.mark.parametrize("m,n", [(77, 300), (45, 5119)])
def test_gram_matvec_integer_construction_is_exact_and_scales(m, n):
    """The reference of the A^T (A x) kernel: small integers, every partial sum below 2^53, so a float64 sum in any order
    is the int64 result; 2^ka A and 2^kx x give 2^(2 ka + kx) times it."""
    rng = np.random.default_rng(m + n)
    A = rng.integers(-3, 4, (m, n)).astype(np.float64)
    x = rng.integers(-3, 4, n).astype(np.float64)
    Ai = A.astype(np.int64)
    want = (Ai.T @ (Ai @ x.astype(np.int64))).astype(np.float64)
    t = np.zeros(m)
    for j in range(n):                                   # sequential in column order, as one lane chain would
        t = t + A[:, j] * x[j]
    y = np.zeros(n)
    for r in range(m):
        y = y + t[r] * A[r]
    assert identical(y, want) and identical(A.T @ (A @ x), want)
    for ka, kx in [(1, 0), (-37, 0), (400, 0), (0, -500)]:
        assert identical((A * p2(ka)).T @ ((A * p2(ka)) @ (x * p2(kx))), np.ldexp(want, 2 * ka + kx))


def test_norm_oracle_scales_exactly():
    rng = np.random.default_rng(8)
    A = away_from_zero(rng, (4097, 45))
    for mode, ks in (("1", (1, -37, 500, -500)), ("inf", (1, -37, 500, -500)), ("fro", (1, -37, 485, -510, 900, -1000))):
        base = do.norm(A, mode)
        for k in ks:
            assert identical(do.norm(A * p2(k), mode), math.ldexp(base, k)), (mode, k)


def test_pagerank_oracle_step_scales_exactly():
    rng = np.random.default_rng(9)
    n = 3000
    src, dst = po.random_graph(n, seed=4)
    L = po.InLinks(*po.link_rows(src, dst, n), n)
    x = 0.5 + 0.5 * rng.random(n)
    base = L.step(x, 0.15)
    for k in (1, -1, 37, -37, 500, -500):
        assert identical(L.step(x * p2(k), 0.15 * p2(k)), np.ldexp(base, k)), k

"""The kernels added after the fp64 edge suite, held to its three exact checks: power-of-two scaling, special values, and
views inside poisoned parents.

  * Scaling: multiplying inputs by powers of two multiplies every product, sum, quotient and square root a linear kernel
    forms by a fixed power of two without changing a significand bit, as long as no intermediate leaves the normal range.
    So the scaled call must give the unscaled call's result, ldexp'ed, bit for bit, whatever the kernel's order.  Each
    scaling test also checks its unscaled call against the kernel's high-precision reference, so a kernel that is wrong in
    a scale-invariant way cannot pass.  The range argument for each is stated beside it.
  * Special values: a NaN or Inf reaches exactly the outputs it should, and every other output keeps its bits.
  * Poisoned parents: operands are views inside NaN-filled parents (odd leading dimensions and views that start 8 bytes
    past a 16-byte boundary among them), outputs views inside sentinel-filled parents.  The result is the packed call's,
    bit for bit, and nothing outside the output view changes.  A kernel that reads one element past a row or column of a
    view, or writes one past it, fails here.
"""
import ctypes as C

import numpy as np
import pytest

from marlin_b200 import _native as nat
from tests import als_oracle as ao
from tests import dms_api_oracle as do
from tests import pagerank_oracle as po
from tests import sparse_oracle as so
from tests import spvec_oracle as sv
from tests.test_gpu_cabi import alloc, download, upload_mat
from tests.test_gpu_fp64_edges import (SENTINEL, _check_out, _out_view, _parent_with, _view_of, cuda, identical,
                                       p2, same, sync, wrap)

pytestmark = pytest.mark.gpu
U_ = 2.0 ** -53


@pytest.fixture(scope="module")
def gpu():
    """The runtime's own context, so C-ABI views and SubMatrix handles can be mixed in one call."""
    import marlin_b200 as mb
    rt = mb.Runtime.get()
    rt.sync_stream()
    return rt.lib, rt.ctx


def away_from_zero(rng, shape, lo=0.5):
    """Random signs times U[lo, 1): every entry has exponent -1, so a scale keeps all of them in a known binade."""
    return np.where(rng.random(shape) < 0.5, -1.0, 1.0) * (lo + (1 - lo) * rng.random(shape))


def ints(rng, shape, lo=-3, hi=3):
    return rng.integers(lo, hi + 1, shape).astype(np.float64)


def _rowshard_nan(A, ld=None, offset=0, fill=np.nan):
    """A (m x n) as a row shard (row r at offset + r * ld) of a device buffer filled with `fill` everywhere else, with two
    more filled doubles after the last row so a 16-byte-aligned span of it reads the fill.  Returns (SubMatrix, buffer)."""
    import torch
    import marlin_b200 as mb
    m, n = A.shape
    ld = max(1, n) if ld is None else ld
    host = np.full(offset + max(m, 1) * ld + 2, fill)
    if m:
        host[offset: offset + m * ld].reshape(m, ld)[:, :n] = A
    buf = torch.from_numpy(host).cuda()
    return mb.SubMatrix(buf=buf, rows=m, cols=n, ld=ld, offset=offset, is_transpose=True), buf


def _outside_untouched(buf, offset, rows, cols, ld, row_major):
    """Every element of the flat parent outside the (rows x cols) view still holds SENTINEL."""
    h = buf.cpu().numpy().copy()
    for i in range(rows if row_major else cols):
        h[offset + i * ld: offset + i * ld + (cols if row_major else rows)] = SENTINEL
    return bool(np.all(h == SENTINEL))


def _vec_in(gpu, v, fill, row=False):
    """v as an fp64 vector view inside a parent filled with `fill`: a column (n x 1, unit stride, offset 1 + ld) or a row
    (1 x n, element stride 3, odd).  Returns (tensor, handle, (rows, cols, ld, offset))."""
    v = np.asarray(v, dtype=np.float64)
    if row:
        X, ld, r0, c0, total = v[None, :], 3, 1, 2, v.size + 4
    else:
        X, ld, r0, c0, total = v[:, None], v.size + 3, 1, 1, 3
    P, off = _parent_with(X, ld, r0, c0, total, fill=fill)
    t = cuda(P)
    return t, wrap(gpu, t, X.shape[0], X.shape[1], ld, off), (X.shape[0], X.shape[1], ld, off)


# =============================================================================== A^T A x (gm_tile_kernel / gm_fold_kernel)
def _gmv(gpu, A_handle, xh, yh, accumulate=False):
    lib, ctx = gpu
    nat.check(lib.mb_block_gram_matvec(ctx, A_handle, xh, yh, int(accumulate)))
    sync(gpu)


def _gm_packed(gpu, blk, x, y0=None):
    n = x.size
    hx, hy = upload_mat(gpu, x[:, None]), upload_mat(gpu, (np.zeros(n) if y0 is None else y0)[:, None])
    _gmv(gpu, blk.handle(), hx, hy, y0 is not None)
    return download(gpu, hy, n, 1).reshape(-1)


# (m, n): resident rows of 16 (m = 77 leaves a ragged last tile), one resident row of 5118 columns per tile, the first wide
# shape (8-row tiles, pieces of 638 columns), and a wide shape with a ragged last piece
GM_SHAPES = [(77, 300), (45, 5118), (45, 5119), (77, 6000)]
# Views: packed, an odd ld starting 8 bytes past a 16-byte boundary (every other row is then 8 bytes off), an even ld
# padded by two, an odd ld starting on a boundary.
GM_VIEWS = [(0, 0), (3, 1), (2, 1), (1, 0)]


@pytest.mark.parametrize("m,n", GM_SHAPES)
def test_gram_matvec_exact_integers_in_nan_parents(gpu, m, n):
    """The reference: integers whose every partial sum fits in 53 bits are summed without rounding in any order, so the
    kernel must give int64 A^T (A x) exactly, on every view; the NaN padding around each row reaches a sum if the kernel
    takes a double from outside the row."""
    rng = np.random.default_rng(m * 7 + n)
    A, x = ints(rng, (m, n)), ints(rng, n)
    Ai = A.astype(np.int64)
    want = (Ai.T @ (Ai @ x.astype(np.int64))).astype(np.float64)
    for extra, off in GM_VIEWS:
        blk, _ = _rowshard_nan(A, ld=n + extra, offset=off)
        assert np.array_equal(_gm_packed(gpu, blk, x), want), (extra, off)


# (ka, kx): A -> 2^ka A, x -> 2^kx x gives y -> 2^(2 ka + kx) y.  Entries of magnitude [0.5, 1): products >= 2^-2, every
# nonzero partial sum of t_r = a_r . x is a multiple of 2^-55 and below 2^13, every nonzero partial sum of y a multiple of
# 2^-110 and below 2^30.  So t stays within [2^(-55 + ka + kx), 2^(13 + ka + kx)] and y within [2^(-110 + s), 2^(30 + s)],
# s = 2 ka + kx: normal for every pair below (|s| <= 800, |ka + kx| <= 500).
GM_SCALES = [(1, 0), (-1, 0), (37, 0), (-37, 0), (0, 500), (0, -500), (400, 0), (-400, 0), (37, -37)]


@pytest.mark.parametrize("m,n", GM_SHAPES)
def test_gram_matvec_power_of_two_scaling(gpu, m, n):
    rng = np.random.default_rng(m + 3 * n)
    A, x, y0 = away_from_zero(rng, (m, n)), away_from_zero(rng, n), away_from_zero(rng, n)
    blk, _ = _rowshard_nan(A, ld=n + 3, offset=1)
    base = _gm_packed(gpu, blk, x)
    base_acc = _gm_packed(gpu, blk, x, y0)
    assert identical(base_acc, y0 + base)                                    # y0 is added once, after the sum
    ref = A.T @ (A @ x)
    assert np.all(np.abs(base - ref) <= 2 * (m + n) * U_ * (np.abs(A).T @ (np.abs(A) @ np.abs(x))))
    for ka, kx in GM_SCALES:
        s = 2 * ka + kx
        sblk, _ = _rowshard_nan(A * p2(ka), ld=n + 3, offset=1)
        assert identical(_gm_packed(gpu, sblk, x * p2(kx)), np.ldexp(base, s)), (ka, kx)
        assert identical(_gm_packed(gpu, sblk, x * p2(kx), y0 * p2(s)), np.ldexp(base_acc, s)), (ka, kx)


@pytest.mark.parametrize("m,n", [(77, 300), (45, 5119)])
def test_gram_matvec_views_in_poisoned_parents(gpu, m, n):
    """x as a column and as a strided row inside NaN parents, y as a column and as a strided row inside sentinel parents,
    with and without accumulate: the packed call's bits, and nothing outside y written."""
    lib, ctx = gpu
    rng = np.random.default_rng(n)
    A, x, y0 = rng.standard_normal((m, n)), rng.standard_normal(n), rng.standard_normal(n)
    packed = _gm_packed(gpu, _rowshard_nan(A)[0], x)
    packed_acc = _gm_packed(gpu, _rowshard_nan(A)[0], x, y0)
    blk, _ = _rowshard_nan(A, ld=n + 3, offset=1)
    for xrow in (False, True):
        tx, hx, _ = _vec_in(gpu, x, np.nan, row=xrow)
        for yrow in (False, True):
            shape = (1, n) if yrow else (n, 1)
            ty, hy, meta = _out_view(gpu, *shape, pad=(2, 3, 1, 1) if yrow else (4, 3, 2, 1))
            _gmv(gpu, blk.handle(), hx, hy)
            assert identical(_check_out(ty, *shape, meta).reshape(-1), packed), (xrow, yrow)
            nat.check(lib.mb_block_copy(ctx, upload_mat(gpu, y0.reshape(shape)), hy))
            _gmv(gpu, blk.handle(), hx, hy, accumulate=True)
            assert identical(_check_out(ty, *shape, meta).reshape(-1), packed_acc), (xrow, yrow)


# =============================================================================== norms (norm_tile_kernel + folds)
def _norm(gpu, h, kind, col=None):
    """mb_block_norm: out[0] is the 1- or inf-norm, or (asml, amed, abig), Blue's three device accumulators, for FRO."""
    lib, ctx = gpu
    out = np.zeros(3)
    nat.check(lib.mb_block_norm(ctx, h, kind, col, out.ctypes.data_as(nat.c_dp)))
    return out


def _norm_views(gpu, A):
    """A as a row shard (lanes along the columns) with an odd ld starting 8 bytes past a 16-byte boundary, and as a
    column-major view (lanes along the rows) with an odd ld, both inside NaN parents."""
    m, n = A.shape
    rowshard, buf = _rowshard_nan(A, ld=n + 3, offset=1)
    t, colmajor = _view_of(gpu, A, 0, pad=(5 if m % 2 == 0 else 4, 3, 1, 2))
    return [("row shard", rowshard.handle(), (rowshard, buf)), ("column-major", colmajor, t)]


def _one(gpu, h, n):
    col = alloc(gpu, n, 1)
    out = _norm(gpu, h, nat.MB_NORM_ONE, col)
    return out[0], download(gpu, col, n, 1).reshape(-1)


NORM_SHAPES = [(4097, 45), (8195, 33), (100, 64)]              # across NORM_CHUNK = 4096; n not a multiple of 32


@pytest.mark.parametrize("m,n", NORM_SHAPES)
def test_norm_exact_integers_and_sequential_inf(gpu, m, n):
    """The references: on integers every column sum and every sum of squares is exact in any order, so the 1-norm, the
    column sums and the middle accumulator are the int64 ones (and the small and big accumulators stay 0.0); the inf-norm
    is the left fold of each row in column order, bit for bit, on random data."""
    rng = np.random.default_rng(m + n)
    A = ints(rng, (m, n), -8, 8)
    R = rng.standard_normal((m, n)) * 10.0 ** rng.integers(-3, 4, (m, n))
    Ai = np.abs(A.astype(np.int64))
    for name, h, _keep in _norm_views(gpu, A):
        best, col = _one(gpu, h, n)
        assert np.array_equal(col, Ai.sum(axis=0).astype(np.float64)) and best == Ai.sum(axis=0).max(), name
        assert np.array_equal(_norm(gpu, h, nat.MB_NORM_FRO), [0.0, float((Ai * Ai).sum()), 0.0]), name
    for name, h, _keep in _norm_views(gpu, R):
        assert identical(_norm(gpu, h, nat.MB_NORM_INF)[0], do.norm(R, "inf")), name


@pytest.mark.parametrize("m,n", NORM_SHAPES)
def test_norm_power_of_two_scaling(gpu, m, n):
    """1 and inf: sums of |a| with |a| in [0.5, 1) lie in [2^-1, 2^14], so 2^k A with |k| <= 500 gives 2^k times every
    column sum and both norms.  Frobenius: 2^k A keeps every entry in Blue's middle band [2^-511, 2^486] for
    k in [-510, 485], where the accumulators are (0, sum a^2, 0): the middle one scales by 4^k (its terms lie in
    [2^-1022, 2^970]) and the norm, its square root, by 2^k."""
    import marlin_b200 as mb
    rng = np.random.default_rng(3 * m + n)
    A = away_from_zero(rng, (m, n))
    for name, h, _keep in _norm_views(gpu, A):
        best, col = _one(gpu, h, n)
        inf = _norm(gpu, h, nat.MB_NORM_INF)[0]
        fro = _norm(gpu, h, nat.MB_NORM_FRO)
        assert fro[0] == 0.0 and fro[2] == 0.0 and fro[1] > 0.0, name
        assert abs(fro[1] - np.sum(A * A)) <= m * n * U_ * np.sum(A * A)                      # the reference, rounded
        assert abs(best - do.norm(A, "1")) <= m * U_ * best and identical(inf, do.norm(A, "inf"))
        for k in (1, -1, 37, -37, 500, -500):
            _, hs, _keep2 = [v for v in _norm_views(gpu, A * p2(k)) if v[0] == name][0]
            sbest, scol = _one(gpu, hs, n)
            assert identical(scol, np.ldexp(col, k)) and identical(sbest, np.ldexp(best, k)), (name, k)
            assert identical(_norm(gpu, hs, nat.MB_NORM_INF)[0], np.ldexp(inf, k)), (name, k)
        for k in (1, -1, 37, -37, 485, -510):
            _, hs, _keep2 = [v for v in _norm_views(gpu, A * p2(k)) if v[0] == name][0]
            assert identical(_norm(gpu, hs, nat.MB_NORM_FRO), [0.0, np.ldexp(fro[1], 2 * k), 0.0]), (name, k)
    base = mb.DenseVecMatrix(ids=np.arange(m), data=_rowshard_nan(A)[0], nRows=m, nCols=n).norm("fro")
    for k in (1, -37, 485, -510):
        got = mb.DenseVecMatrix(ids=np.arange(m), data=_rowshard_nan(A * p2(k))[0], nRows=m, nCols=n).norm("fro")
        assert identical(got, np.ldexp(base, k)), k


def test_frobenius_within_rounding_across_blue_bands(gpu):
    """Scales that move entries out of the middle band (k > 485 or k < -510 for entries of magnitude [0.5, 1)), and rows
    spread over all three bands at once: the norm stays within (m n + 8) u of the exact one (sqrt of the scaled sum of
    squares, scaled back), as dnrm2's bound states."""
    import marlin_b200 as mb
    m, n = 4097, 45
    rng = np.random.default_rng(77)
    A = away_from_zero(rng, (m, n))
    exact = do.norm(A, "fro")
    bound = (m * n + 8) * U_
    for k in (480, 486, 487, 500, 900, -509, -511, -512, -600, -1000):
        got = mb.DenseVecMatrix(ids=np.arange(m), data=_rowshard_nan(A * p2(k), ld=n + 3, offset=1)[0], nRows=m,
                                nCols=n).norm("fro")
        assert abs(got - np.ldexp(exact, k)) <= bound * np.ldexp(exact, k), k
    e = rng.choice([-600, -520, -300, 0, 300, 490, 500], size=m)
    S = A * np.exp2(e.astype(float))[:, None]
    got = mb.DenseVecMatrix(ids=np.arange(m), data=_rowshard_nan(S, ld=n + 3, offset=1)[0], nRows=m, nCols=n).norm("fro")
    assert abs(got - do.norm(S, "fro")) <= bound * do.norm(S, "fro")


def test_norm_column_sums_into_views_in_poisoned_parents(gpu):
    """The column sums as a column and as a strided row inside sentinel parents: the packed call's bits, nothing else
    written; the norms of the poisoned views are the packed block's."""
    lib, ctx = gpu
    m, n = 4097, 45
    A = np.random.default_rng(5).standard_normal((m, n))
    hp = upload_mat(gpu, A)
    best, col = _one(gpu, hp, n)
    for name, h, _keep in _norm_views(gpu, A):
        for row in (False, True):
            shape = (1, n) if row else (n, 1)
            t, hc, meta = _out_view(gpu, *shape, pad=(2, 3, 1, 1) if row else (4, 3, 2, 1))
            out = _norm(gpu, h, nat.MB_NORM_ONE, hc)
            sync(gpu)
            assert identical(_check_out(t, *shape, meta).reshape(-1), col) and identical(out[0], best), (name, row)
        for kind in (nat.MB_NORM_INF, nat.MB_NORM_FRO):
            assert identical(_norm(gpu, h, kind), _norm(gpu, hp, kind)), (name, kind)


def test_norm_nan_and_inf_reach_only_their_column_sums(gpu):
    m, n = 4100, 45
    rng = np.random.default_rng(6)
    A = rng.standard_normal((m, n))
    clean = _one(gpu, upload_mat(gpu, A), n)[1]
    A[4097, 3], A[10, 40] = np.nan, -np.inf
    for name, h, _keep in _norm_views(gpu, A):
        best, col = _one(gpu, h, n)
        assert np.isnan(col[3]) and np.isposinf(col[40]) and np.isnan(best), name
        rest = np.ones(n, bool)
        rest[[3, 40]] = False
        assert identical(col[rest], clean[rest]), name


# =============================================================================== ALS (als_kernel<G, EPT, SOLVE>)
def _als_side(L):
    import marlin_b200 as mb
    rt = mb.Runtime.get()
    rt.sync_stream()
    return rt, L.to_device(rt.device)


def _als_assemble(L, Yblk, lam, implicit=False, alpha=1.0, yty=None):
    import torch
    from tests.test_gpu_als import _rows_block
    rt, (side, _keep) = _als_side(L)
    r = Yblk.cols
    A = torch.full((L.n * (r * (r + 1) // 2),), float("nan"), dtype=torch.float64, device=rt.device)
    b = torch.full((L.n * r,), float("nan"), dtype=torch.float64, device=rt.device)
    G = _rows_block(yty) if yty is not None else None
    nat.check(rt.lib.mb_als_normal_equations(rt.ctx, C.byref(side), Yblk.handle(), lam, alpha, int(implicit),
                                             G.handle() if G is not None else None, C.c_void_p(A.data_ptr()),
                                             C.c_void_p(b.data_ptr())))
    return A.cpu().numpy().reshape(L.n, -1), b.cpu().numpy().reshape(L.n, r)


def _als_solve(L, Yblk, lam, implicit=False, alpha=1.0, yty=None, ld=None, offset=0):
    """x_u for every entity, written into a row-major view (ld, offset) of a SENTINEL-filled parent whose view starts as
    SENTINEL too.  Returns (X, parent untouched outside the view, error or None)."""
    from tests.test_gpu_als import _rows_block
    rt, (side, _keep) = _als_side(L)
    r = Yblk.cols
    ld = r if ld is None else ld
    Xblk, buf = _rowshard_nan(np.full((L.n, r), SENTINEL), ld=ld, offset=offset, fill=SENTINEL)
    G = _rows_block(yty) if yty is not None else None
    err = None
    try:
        nat.check(rt.lib.mb_als_update(rt.ctx, C.byref(side), Yblk.handle(), lam, alpha, int(implicit),
                                       G.handle() if G is not None else None, Xblk.handle()))
    except nat.MarlinError as e:
        err = e
    rt.synchronize()
    return Xblk.toBreeze(), _outside_untouched(buf, offset, L.n, r, ld, True), err


def _als_case(rank, seed, implicit=False):
    from tests.test_gpu_als import _data, _links
    rows, cols, vals = _data(40, 60, 2400, seed, heavy=1500, signed=implicit)
    L = _links(rows, cols, vals, 3, 4)
    Y = away_from_zero(np.random.default_rng(seed), (len(np.unique(cols)), rank))
    return L, ao.links(rows, cols, vals, 3, 4), Y


ALS_RANKS = [10, 11, 32, 33, 50, 51]                     # both sides of the warp/CTA template buckets


@pytest.mark.parametrize("implicit", [False, True])
@pytest.mark.parametrize("rank", ALS_RANKS)
def test_als_power_of_two_scaling(rank, implicit):
    """Y -> 2^k Y with lambda -> 4^k lambda (and YtY -> 4^k YtY when implicit) gives A -> 4^k A and b -> 2^k b exactly:
    every term of A is a product of two entries of Y (times c - 1, unscaled) and n_u lambda, every term of b a rating (or
    c) times one.  The Cholesky pivots' square roots then scale by 2^k exactly, every division and update by a fixed power
    too, so x -> 2^-k x.  Entries of Y in [0.5, 1): A's terms lie in [2^-2, 2^4], the solve's intermediates far inside
    [2^-400, 2^400], so |k| <= 250 keeps all of them normal.  The unscaled assembly is the oracle's bit for bit and the
    unscaled solve within the kappa(A) bound of tests/test_gpu_als.py."""
    from tests.test_gpu_als import _rows_block, _solve_bound
    L, Lo, Y = _als_case(rank, rank + 100 * implicit, implicit)
    lam, alpha = 0.05, 0.37
    yty = ao.gramian(Y) if implicit else None
    A0, b0 = _als_assemble(L, _rows_block(Y), lam, implicit, alpha, yty)
    Ar, br = ao.assemble(Lo, Y, lam, implicit=implicit, alpha=alpha, yty=yty)
    assert identical(A0, Ar) and identical(b0, br)
    X0, _, err = _als_solve(L, _rows_block(Y), lam, implicit, alpha, yty)
    assert err is None
    if not implicit:
        for p in range(0, L.n, 7):
            _, x_cho, bound = _solve_bound(Ar[p], br[p], rank)
            assert np.abs(X0[p] - x_cho).max() <= bound, p
    for k in (1, -1, 37, -37, 250, -250):
        Ys, ls, ys = Y * p2(k), lam * p2(2 * k), None if yty is None else yty * p2(2 * k)
        A, b = _als_assemble(L, _rows_block(Ys), ls, implicit, alpha, ys)
        assert identical(A, np.ldexp(A0, 2 * k)) and identical(b, np.ldexp(b0, k)), k
        X, _, err = _als_solve(L, _rows_block(Ys), ls, implicit, alpha, ys)
        assert err is None and identical(X, np.ldexp(X0, -k)), k


@pytest.mark.parametrize("rank", [11, 33])
def test_als_views_in_poisoned_parents(rank):
    """Y as a row shard with an odd ld, 8 bytes past a 16-byte boundary, in a NaN parent; X as a strided view of a
    sentinel parent: the packed call's bits, and nothing outside X written."""
    from tests.test_gpu_als import _rows_block
    L, _, Y = _als_case(rank, 7 * rank)
    A0, b0 = _als_assemble(L, _rows_block(Y), 0.05)
    X0, _, _ = _als_solve(L, _rows_block(Y), 0.05)
    Yv, _keep = _rowshard_nan(Y, ld=rank + 3, offset=1)
    A, b = _als_assemble(L, Yv, 0.05)
    assert identical(A, A0) and identical(b, b0)
    X, untouched, err = _als_solve(L, Yv, 0.05, ld=rank + 5, offset=3)
    assert err is None and untouched and identical(X, X0)


def _tri_mask(r, c):
    """Packed lower triangle (row-major): the elements in row or column c."""
    i = np.concatenate([np.full(k + 1, k) for k in range(r)])
    j = np.concatenate([np.arange(k + 1) for k in range(r)])
    return (i == c) | (j == c)


@pytest.mark.parametrize("rank", [11, 33])
def test_als_nan_in_one_partner_row_poisons_only_its_raters(rank):
    """Y[p, c] = NaN: for the entities that rated partner p, A's row and column c and b[c] become NaN and nothing else
    changes; every other entity keeps its bits.  The solve stops at pivot c for exactly those entities: the lowest of
    their ids is named, their rows of X stay unwritten, and every other row is the clean solve's."""
    from tests.test_gpu_als import _rows_block
    L, _, Y = _als_case(rank, 3 * rank)
    A0, b0 = _als_assemble(L, _rows_block(Y), 0.05)
    X0, _, _ = _als_solve(L, _rows_block(Y), 0.05)
    counts = np.bincount(L.partners[:L.offsets[L.n]], minlength=Y.shape[0])
    p, c = int(np.argsort(counts)[len(counts) // 2]), rank // 2          # a partner rated by a few entities
    raters = np.array([(L.partners[L.offsets[u]:L.offsets[u + 1]] == p).any() for u in range(L.n)])
    assert 0 < raters.sum() < L.n
    Yn = Y.copy()
    Yn[p, c] = np.nan
    A, b = _als_assemble(L, _rows_block(Yn), 0.05)
    mask = _tri_mask(rank, c)
    assert identical(A[~raters], A0[~raters]) and identical(b[~raters], b0[~raters])
    assert np.all(np.isnan(A[raters][:, mask])) and identical(A[raters][:, ~mask], A0[raters][:, ~mask])
    assert np.all(np.isnan(b[raters][:, c]))
    keep = np.ones(rank, bool)
    keep[c] = False
    assert identical(b[raters][:, keep], b0[raters][:, keep])
    X, untouched, err = _als_solve(L, _rows_block(Yn), 0.05, ld=rank + 1, offset=1)
    assert err is not None and f"entity {int(L.ids[:L.n][raters].min())} are not positive definite" in str(err)
    assert untouched and np.all(X[raters] == SENTINEL) and identical(X[~raters], X0[~raters])


# =============================================================================== sparse blocks (dense_sparse, sparse_dense, spgemm)
_SP_KEEP = []


def _sp(gpu, S):
    lib, ctx = gpu
    rows, cols, cp, ri, va = S
    cp, ri, va = (np.ascontiguousarray(a, dt) for a, dt in ((cp, np.int32), (ri, np.int32), (va, np.float64)))
    h = nat.c_sp()
    nat.check(lib.mb_sparse_upload(ctx, rows, cols, cp.ctypes.data, ri.ctypes.data, va.ctypes.data, C.byref(h)))
    _SP_KEEP.append(h)
    return h


def _scaled(S, k):
    return S[0], S[1], S[2], S[3], S[4] * p2(k)


def _sparse_product(gpu, kind, left, right, m, n, C0=None, cview=None):
    """kind 'ds': dense left x sparse right; 'sd': sparse left x dense right; 'ss': sparse x sparse.  Dense operands are
    host arrays (uploaded packed) or handles; the result goes into a packed block, or into `cview` = (tensor, handle,
    meta) of a sentinel parent.  C0: accumulate onto it."""
    lib, ctx = gpu
    if cview is None:
        hc = upload_mat(gpu, C0) if C0 is not None else alloc(gpu, m, n)
    else:
        hc = cview[1]
        if C0 is not None:
            nat.check(lib.mb_block_copy(ctx, upload_mat(gpu, C0), hc))
    dense = lambda X: upload_mat(gpu, X) if isinstance(X, np.ndarray) else X
    acc = int(C0 is not None)
    if kind == "ds":
        nat.check(lib.mb_spmm_dense_sparse(ctx, dense(left), _sp(gpu, right), hc, acc))
    elif kind == "sd":
        nat.check(lib.mb_spmm_sparse_dense(ctx, _sp(gpu, left), dense(right), hc, acc))
    else:
        nat.check(lib.mb_spgemm_dense_out(ctx, _sp(gpu, left), _sp(gpu, right), hc, acc))
    sync(gpu)
    if cview is None:
        return download(gpu, hc, m, n)
    return _check_out(cview[0], m, n, cview[2])


def _sparse_case(kind, seed):
    """m = 1100 rows, so the sparse x sparse kernel splits each column into two chunks of SPG_CHUNK = 1024 rows."""
    rng = np.random.default_rng(seed)
    m, k, n = 1100, 300, 70
    vals = lambda shape: away_from_zero(rng, shape)
    csc = lambda r, c, d: so.csc_from_dense_pattern(vals((r, c)), rng.random((r, c)) < d)
    if kind == "ds":
        left, right, ref = vals((m, k)), csc(k, n, 0.05), so.mult_dense_sparse
    elif kind == "sd":
        left, right, ref = csc(m, k, 0.05), vals((k, n)), so.mult_sparse_dense
    else:
        left, right, ref = csc(m, k, 0.05), csc(k, n, 0.05), so.spgemm
    return left, right, ref, vals((m, n)), m, n


def _scale_operand(X, k):
    return X * p2(k) if isinstance(X, np.ndarray) else _scaled(X, k)


@pytest.mark.parametrize("kind", ["ds", "sd", "ss"])
def test_sparse_products_power_of_two_scaling(gpu, kind):
    """Left -> 2^a left, right -> 2^b right, C -> 2^(a+b) C gives 2^(a+b) times the product and the accumulated sum.
    Values of magnitude [0.5, 1): products >= 2^-2, nonzero partial sums multiples of 2^-55 and below 2^10, so
    |a + b| <= 900 with |a|, |b| <= 500 keeps every one normal.  The unscaled product, and C + product when
    accumulating, are the reference loops' bits (tests/sparse_oracle.py)."""
    left, right, ref, C0, m, n = _sparse_case(kind, ord(kind[0]) + ord(kind[1]))
    base = _sparse_product(gpu, kind, left, right, m, n)
    base_acc = _sparse_product(gpu, kind, left, right, m, n, C0=C0)
    want = ref(left, right)
    assert same(base, want) and same(base_acc, C0 + want)                 # C is added once, after the whole sum
    for a, b in [(1, 0), (0, -1), (37, 0), (0, -37), (500, -1), (-500, 1), (450, 450), (-450, -450)]:
        L, R = _scale_operand(left, a), _scale_operand(right, b)
        assert identical(_sparse_product(gpu, kind, L, R, m, n), np.ldexp(base, a + b)), (a, b)
        assert identical(_sparse_product(gpu, kind, L, R, m, n, C0=C0 * p2(a + b)), np.ldexp(base_acc, a + b)), (a, b)


@pytest.mark.parametrize("kind", ["ds", "sd", "ss"])
def test_sparse_products_views_in_poisoned_parents(gpu, kind):
    """The dense operand as a view (stored as is, or transposed) inside a NaN parent; C as a view inside a sentinel
    parent, overwritten and accumulated onto (these kernels read C then): the packed call's bits, nothing else written."""
    left, right, _, C0, m, n = _sparse_case(kind, 11 + len(kind))
    want = _sparse_product(gpu, kind, left, right, m, n)
    want_acc = _sparse_product(gpu, kind, left, right, m, n, C0=C0)
    for trans in (0, 1):
        keep = []
        if kind == "ds":
            keep.append(_view_of(gpu, left, trans))
            left_v, right_v = keep[-1][1], right
        elif kind == "sd":
            keep.append(_view_of(gpu, right, trans))
            left_v, right_v = left, keep[-1][1]
        else:
            left_v, right_v = left, right
        cv = _out_view(gpu, m, n)
        assert identical(_sparse_product(gpu, kind, left_v, right_v, m, n, cview=cv), want), trans
        assert identical(_sparse_product(gpu, kind, left_v, right_v, m, n, C0=C0, cview=cv), want_acc), trans


@pytest.mark.parametrize("kind", ["ds", "sd"])
def test_sparse_products_nan_and_inf_reach_only_their_outputs(gpu, kind):
    """A NaN and an Inf in the dense operand reach exactly the outputs whose sums take them (the reference loops say which;
    Inf * a negative value is -Inf, an Inf meeting the opposite Inf is NaN), and every other output keeps its bits."""
    left, right, ref, C0, m, n = _sparse_case(kind, 23 + len(kind))
    clean = _sparse_product(gpu, kind, left, right, m, n)
    if kind == "ds":                                   # rows k of the sparse right operand that hold values
        k0, k1 = int(right[3][0]), int(right[3][-1])
        left = left.copy()
        left[5, k0], left[1050, k1] = np.nan, np.inf
    else:                                              # columns k of the sparse left operand that hold values
        k0, k1 = [int(k) for k in np.flatnonzero(np.diff(left[2]))[[0, -1]]]
        right = right.copy()
        right[k0, 5], right[k1, 60] = np.nan, -np.inf
    got = _sparse_product(gpu, kind, left, right, m, n, C0=C0)
    want = C0 + ref(left, right)
    assert same(got, want)
    hit = ~np.isfinite(want)
    assert hit.any() and identical(got[~hit], (C0 + clean)[~hit])


# =============================================================================== SparseVecMatrix products (spvec_*, float)
def _spvec(A, B, m, K, n):
    from tests.test_gpu_spvec import _coo, _mat
    return _coo(_mat(A, m, K).multiplySparse(_mat(B, K, n)))


def _spvec_bin_case():
    """tests/test_gpu_spvec.py's bin case (one row at every count around MB_SPVEC_WARP_BOUND and MB_SPVEC_CTA_BOUND, rows
    far beyond the CTA hash, an empty row) with every value of magnitude [0.5, 1)."""
    from tests.test_gpu_spvec import _bin_case
    A, B, m, K, n = _bin_case(1)
    rng = np.random.default_rng(2)
    A = [(i, ix, away_from_zero(rng, len(ix))) for i, ix, _ in A]
    B = [(k, ix, away_from_zero(rng, len(ix))) for k, ix, _ in B]
    return A, B, m, K, n


def _scale_rows(rows, k):
    return [(i, ix, np.asarray(v) * p2(k)) for i, ix, v in rows]


def test_spvec_power_of_two_scaling_in_every_bin():
    """(2^a A)(2^b B) in float: f32(2^a v) = 2^a f32(v) while normal, every product is 2^(a+b) times the unscaled float
    product, every sum too.  Products lie in [2^-2, 1) and are multiples of 2^-25, every nonzero partial sum is a multiple
    of 2^-25 below 2^17, so |a + b| <= 100 with |a|, |b| <= 60 keeps them in float's normal range [2^-126, 2^128).  The
    unscaled product is the oracle's fixed-order float sums bit for bit."""
    from tests.test_gpu_spvec import _assert_bits
    A, B, m, K, n = _spvec_bin_case()
    base = _spvec(A, B, m, K, n)
    _assert_bits(base, sv.multiply_sparse(A, B))
    for a, b in [(1, 0), (0, -1), (37, 0), (0, -37), (37, -37), (60, 40), (-60, -40), (60, -60)]:
        r, c, v = _spvec(_scale_rows(A, a), _scale_rows(B, b), m, K, n)
        assert np.array_equal(r, base[0]) and np.array_equal(c, base[1])
        assert np.array_equal(v.view(np.uint32), np.ldexp(base[2], a + b).astype(np.float32).view(np.uint32)), (a, b)


def test_spvec_scaling_out_of_float_range_matches_the_oracle():
    """Past float's normal range the result is no longer the scaled one: products round to subnormals or overflow to Inf.
    The fixed-order oracle still gives every bit, so the rows of every bin must follow it there too."""
    from tests.test_gpu_spvec import _assert_bits
    A, B, m, K, n = _spvec_bin_case()
    for a, b in [(100, 28), (-100, -40), (64, 63)]:
        As, Bs = _scale_rows(A, a), _scale_rows(B, b)
        _assert_bits(_spvec(As, Bs, m, K, n), sv.multiply_sparse(As, Bs))


def test_spvec_float_overflow_stays_in_its_entry():
    """One product that overflows float (2^100 * 2^30 * [0.25, 1) >= 2^128) makes its C(i, j) +-Inf; every other entry,
    the rest of row i included, keeps the bits it has without that product's overflow."""
    from tests.test_gpu_spvec import _assert_bits
    A, B, m, K, n = _spvec_bin_case()
    t, k0 = next((t, int(k)) for t, (_, ix, _) in enumerate(A) for k in ix if 5000 <= k < 6000)   # a B row of 64
    B = [(k, ix, np.asarray(v) * (p2(30) if k == k0 else 1.0)) for k, ix, v in B]
    i, ix, v = A[t]
    hot = list(ix).index(k0)
    clean = _spvec(A, B, m, K, n)
    v = np.asarray(v).copy()
    v[hot] *= p2(100)
    Ahot = A[:t] + [(i, ix, v)] + A[t + 1:]
    got = _spvec(Ahot, B, m, K, n)
    _assert_bits(got, sv.multiply_sparse(Ahot, B))
    targets = set(int(j) for j in B[[k for k, _, _ in B].index(k0)][1])
    inf = (got[0] == i) & np.isin(got[1], list(targets))
    assert np.all(np.isinf(got[2][inf])) and not np.isinf(got[2][~inf]).any()
    assert np.array_equal(got[2][~inf].view(np.uint32), clean[2][~inf].view(np.uint32))


# =============================================================================== Schur update (grouped DMMA, then subtract)
def _dblk(a, ld=None, offset=0, fill=np.nan):
    """A column-major device block holding a at (ld, offset) inside a parent filled with `fill`."""
    import torch
    import marlin_b200 as mb
    m, n = a.shape
    ld = ld or max(1, m)
    host = np.full(offset + ld * n + 2, fill)
    host[offset: offset + ld * n].reshape(n, ld)[:, :m] = a.T
    buf = torch.from_numpy(host).cuda()
    return mb.SubMatrix(buf=buf, rows=m, cols=n, ld=ld, offset=offset), buf


def _schur(entries):
    from marlin_b200.matrix.factorizations import schur_update
    schur_update(entries)


# Trailing-update grids of tests/test_gpu_factor_dist.py: 9 x 9 entries (more than the 64 entries of one grouped launch)
# and 40 x 2 (more than its 32 distinct A operands), with shared row operands X_r and column operands Y_c.
SCHUR_GRIDS = [(9, 9, 64), (40, 2, 32)]


def _schur_grid(rows, cols, s, X, Y, Cs, **view):
    """C_rc -= X_r Y_c over the grid; X, Y, Cs host arrays.  Returns the C results."""
    xb = [_dblk(x, **view) for x in X]
    yb = [_dblk(y, **view) for y in Y]
    cb = {key: _dblk(c) for key, c in Cs.items()}
    _schur([(cb[(r, c)][0], xb[r][0], yb[c][0]) for r in range(rows) for c in range(cols)])
    return {key: b.toBreeze() for key, (b, _) in cb.items()}


@pytest.mark.parametrize("rows,cols,s", SCHUR_GRIDS)
def test_schur_update_power_of_two_scaling(rows, cols, s):
    """X -> 2^a X, Y -> 2^b Y, C -> 2^(a+b) C gives 2^(a+b) (C - X Y) bit for bit.  Entries of magnitude [0.5, 1): every
    product >= 2^-2, every nonzero partial sum a multiple of 2^-55 below 2^8, so |a + b| <= 900 with |a|, |b| <= 500 keeps
    them normal.  The reference: on integers the update is exact, so it is int64 C - X Y."""
    rng = np.random.default_rng(rows * 10 + cols)
    Xi = [ints(rng, (s, s), -4, 4) for _ in range(rows)]
    Yi = [ints(rng, (s, s), -4, 4) for _ in range(cols)]
    Ci = {(r, c): ints(rng, (s, s), -4, 4) for r in range(rows) for c in range(cols)}
    got = _schur_grid(rows, cols, s, Xi, Yi, Ci)
    for (r, c), v in got.items():
        want = Ci[(r, c)].astype(np.int64) - Xi[r].astype(np.int64) @ Yi[c].astype(np.int64)
        assert np.array_equal(v, want.astype(np.float64)), (r, c)
    X = [away_from_zero(rng, (s, s)) for _ in range(rows)]
    Y = [away_from_zero(rng, (s, s)) for _ in range(cols)]
    Cs = {(r, c): away_from_zero(rng, (s, s)) for r in range(rows) for c in range(cols)}
    base = _schur_grid(rows, cols, s, X, Y, Cs)
    for (r, c), v in base.items():
        assert np.all(np.abs(v - (Cs[(r, c)] - X[r] @ Y[c])) <= 2 * (s + 1) * U_ * (np.abs(Cs[(r, c)]) + np.abs(X[r]) @ np.abs(Y[c])))
    for a, b in [(1, 0), (0, -1), (37, 0), (0, -37), (37, -37), (500, -500), (450, 450), (-450, -450)]:
        got = _schur_grid(rows, cols, s, [x * p2(a) for x in X], [y * p2(b) for y in Y],
                          {key: v * p2(a + b) for key, v in Cs.items()})
        for key, v in got.items():
            assert identical(v, np.ldexp(base[key], a + b)), (a, b, key)


@pytest.mark.parametrize("ld_pad,offset", [(2, 2), (1, 1), (3, 0)])
def test_schur_update_views_in_poisoned_parents(ld_pad, offset):
    """Operands inside NaN parents, B also transposed, targets inside sentinel parents.  Every entry gives the bits of
    gemm-then-subtract on the same views, and nothing outside the targets is written.  Even ld on a 16-byte boundary keeps
    the grouped DMMA path, so those entries must also give the packed call's bits; an odd ld, or a view 8 bytes off the
    boundary, takes the per-entry path, whose GEMM may sum in another order."""
    rng = np.random.default_rng(ld_pad * 10 + offset)
    shapes = [(64, 64, 64), (130, 66, 98), (37, 129, 64)]
    packed, viewed, want, parents = [], [], [], []
    for (m, n, k) in shapes:
        a, b, c = away_from_zero(rng, (m, k)), away_from_zero(rng, (k, n)), away_from_zero(rng, (m, n))
        packed.append((_dblk(c)[0], _dblk(a)[0], _dblk(b)[0]))
        av = _dblk(a, ld=m + ld_pad, offset=offset)[0]
        for bv in (_dblk(np.ascontiguousarray(b.T), ld=n + ld_pad, offset=offset)[0].t,
                   _dblk(b, ld=k + ld_pad, offset=offset)[0]):
            cv, cbuf = _dblk(c, ld=m + ld_pad, offset=offset, fill=SENTINEL)
            want.append(cv.subtract(av.multiply(bv)).toBreeze())
            viewed.append((cv, av, bv))
            parents.append((cbuf, offset, m, n, m + ld_pad))
    _schur(packed)
    _schur(viewed)
    for e, (cv, _, _) in enumerate(viewed):
        assert identical(cv.toBreeze(), want[e]), e
        if ld_pad % 2 == 0 and offset % 2 == 0 and shapes[e // 2][0] % 2 == 0:
            assert identical(cv.toBreeze(), packed[e // 2][0].toBreeze()), e
    for buf, off, m, n, ld in parents:
        assert _outside_untouched(buf, off, n, m, ld, True)


# =============================================================================== logistic gradient (lr_grad_tile_kernel)
@pytest.mark.parametrize("m,n", [(100, 129), (100, 385)])            # one read per row / rows streamed twice
def test_lr_gradient_views_in_poisoned_parents(m, n):
    """Row shards with odd ld, 8 bytes past a 16-byte boundary and with a wide ld, and a column-major block, all inside
    NaN parents: the packed shard's bits (m = 100 leaves a ragged last tile of 4 rows)."""
    from tests.test_gpu_lr import _gradient
    rng = np.random.default_rng(m + n)
    A = rng.standard_normal((m, n))
    A[:, 0] = rng.integers(0, 2, m)
    w = rng.standard_normal(n) / np.sqrt(n)
    ref = _gradient(_rowshard_nan(A)[0], w)
    for ld, off in [(n + 1, 1), (n + 3, 1), (n + 2, 2), (n + 9, 3)]:
        assert identical(_gradient(_rowshard_nan(A, ld=ld, offset=off)[0], w), ref), (ld, off)
    assert identical(_gradient(_dblk(A, ld=m + 3, offset=1)[0], w), ref)


@pytest.mark.parametrize("m,n", [(100, 129), (100, 385)])
def test_lr_gradient_inf_feature_reaches_only_its_column(m, n):
    """x_rj = +Inf with w_j > 0 and label 0: the margin is -Inf, exp gives 0 and g_r = 1, exactly what x_rj = 1e300 gives.
    So the gradient's column j becomes +Inf and every other column keeps the bits of the 1e300 run."""
    from tests.test_gpu_lr import _gradient
    rng = np.random.default_rng(2 * m + n)
    A = rng.standard_normal((m, n))
    A[:, 0] = rng.integers(0, 2, m)
    w = rng.standard_normal(n) / np.sqrt(n)
    r, j = 37, n - 2
    A[r, 0], w[j] = 0.0, 0.5
    big = A.copy()
    big[r, j] = 1e300
    want = _gradient(_rowshard_nan(big, ld=n + 1, offset=1)[0], w)
    A[r, j] = np.inf
    got = _gradient(_rowshard_nan(A, ld=n + 1, offset=1)[0], w)
    assert np.isposinf(got[j])
    rest = np.ones(n, bool)
    rest[j] = False
    assert identical(got[rest], want[rest])


# =============================================================================== NeuralNetwork (nn_backprop_kernel, nn_apply_kernel)
def _handles(hs):
    return (nat.c_blk * len(hs))(*[h.value if hasattr(h, "value") else h for h in hs])


def _nn_call(gpu, Xh, XTh, ys, W1h, W2h, scale, outs=None):
    """mb_nn_gradient (outs = (g1, g2, [D1])) or, with outs None, mb_nn_step updating W1h, W2h in place."""
    import marlin_b200 as mb
    from tests.test_gpu_nn import _Labels
    lib, ctx = gpu
    rt = mb.Runtime.get()
    lab = _Labels(rt, ys)
    try:
        rt.sync_stream()
        xt = _handles(XTh) if XTh is not None else None
        if outs is None:
            nat.check(lib.mb_nn_step(ctx, _handles(Xh), xt, lab.array(), len(Xh), W1h, W2h, scale))
        else:
            nat.check(lib.mb_nn_gradient(ctx, _handles(Xh), xt, lab.array(), len(Xh), W1h, W2h, scale, outs[0], outs[1],
                                         _handles(outs[2])))
        sync(gpu)
    finally:
        lab.free()


def _nn_packed(gpu, Xs, ys, W1, W2, scale):
    V, H = W1.shape
    g1, g2, d1 = alloc(gpu, V, H), alloc(gpu, H, 10), [alloc(gpu, len(X), H) for X in Xs]
    _nn_call(gpu, [upload_mat(gpu, X) for X in Xs], [upload_mat(gpu, X.T) for X in Xs], ys, upload_mat(gpu, W1),
             upload_mat(gpu, W2), scale, (g1, g2, d1))
    return download(gpu, g1, V, H), download(gpu, g2, H, 10), [download(gpu, d, len(X), H) for d, X in zip(d1, Xs)]


NN_ROWS, NN_V, NN_H = [1000, 518], 784, 100        # even sizes: the views below keep the grouped path's alignment


def test_nn_gradient_and_step_views_in_poisoned_parents(gpu):
    """X, X^T, W1 and W2 inside NaN parents; dW1, dW2 and every D1 block, and the weights that mb_nn_step updates in
    place, inside sentinel parents: the packed calls' bits, nothing outside the outputs written."""
    from tests.test_gpu_nn import _case
    lib, ctx = gpu
    Xs, ys, W1, W2 = _case(NN_ROWS, NN_V, NN_H, 31)
    want = _nn_packed(gpu, Xs, ys, W1, W2, 0.25)
    keep = [_view_of(gpu, X) for X in Xs] + [_view_of(gpu, np.ascontiguousarray(X.T)) for X in Xs]
    xv, xtv = [k[1] for k in keep[:len(Xs)]], [k[1] for k in keep[len(Xs):]]
    (t1, w1v), (t2, w2v) = _view_of(gpu, W1), _view_of(gpu, W2)
    g1, g2 = _out_view(gpu, NN_V, NN_H), _out_view(gpu, NN_H, 10)
    d1 = [_out_view(gpu, len(X), NN_H) for X in Xs]
    _nn_call(gpu, xv, xtv, ys, w1v, w2v, 0.25, (g1[1], g2[1], [d[1] for d in d1]))
    assert identical(_check_out(g1[0], NN_V, NN_H, g1[2]), want[0])
    assert identical(_check_out(g2[0], NN_H, 10, g2[2]), want[1])
    for d, X, w in zip(d1, Xs, want[2]):
        assert identical(_check_out(d[0], len(X), NN_H, d[2]), w)
    # the update in place: packed weights against weights held as views of sentinel parents
    p1, p2_ = upload_mat(gpu, W1), upload_mat(gpu, W2)
    _nn_call(gpu, [upload_mat(gpu, X) for X in Xs], [upload_mat(gpu, X.T) for X in Xs], ys, p1, p2_, 0.25)
    u1, u2 = _out_view(gpu, NN_V, NN_H), _out_view(gpu, NN_H, 10)
    nat.check(lib.mb_block_copy(ctx, upload_mat(gpu, W1), u1[1]))
    nat.check(lib.mb_block_copy(ctx, upload_mat(gpu, W2), u2[1]))
    _nn_call(gpu, xv, xtv, ys, u1[1], u2[1], 0.25)
    assert identical(_check_out(u1[0], NN_V, NN_H, u1[2]), download(gpu, p1, NN_V, NN_H))
    assert identical(_check_out(u2[0], NN_H, 10, u2[2]), download(gpu, p2_, NN_H, 10))


def test_nn_nan_feature_poisons_its_delta_row_and_the_gradients():
    """A NaN in row r of one block: that row's hidden delta is NaN and every other row of D1, in both blocks, keeps its
    bits; both weight gradients are sums over all rows, so every element of them is NaN."""
    import marlin_b200 as mb
    from tests.test_gpu_nn import _case
    rt = mb.Runtime.get()
    gpu = (rt.lib, rt.ctx)
    Xs, ys, W1, W2 = _case(NN_ROWS, NN_V, NN_H, 32)
    clean = _nn_packed(gpu, Xs, ys, W1, W2, 0.5)
    Xs[1] = Xs[1].copy()
    Xs[1][300, 400] = np.nan
    g1, g2, d1 = _nn_packed(gpu, Xs, ys, W1, W2, 0.5)
    assert np.all(np.isnan(g1)) and np.all(np.isnan(g2))
    assert identical(d1[0], clean[2][0]) and np.all(np.isnan(d1[1][300]))
    rest = np.ones(NN_ROWS[1], bool)
    rest[300] = False
    assert identical(d1[1][rest], clean[2][1][rest])


# =============================================================================== PageRank (pagerank_step_kernel, both bins)
def _bin_bound_graph():
    """tests/test_gpu_pagerank.py's graph with in-degrees on both sides of MB_PAGERANK_LIGHT_BOUND."""
    b = nat.MB_PAGERANK_LIGHT_BOUND
    rng = np.random.default_rng(3)
    n = 8192
    pattern = [0, 1, 2, 31, 32, b - 1, b, b + 1, b + 2, 2 * b, 700, 5000, 0, 1]
    deg = np.array([pattern[t % len(pattern)] if t % 3 else 200 for t in range(n)])
    deg[64:96] = b
    deg[96:128] = b + 1
    src = np.concatenate([rng.choice(n, d, replace=False) for d in deg])
    dst = np.repeat(np.arange(n), deg)
    return n, src, dst


@pytest.fixture(scope="module")
def pr_graph():
    from tests.test_gpu_pagerank import _c_links
    n, src, dst = _bin_bound_graph()
    return n, src, dst, _c_links(n, src, dst), po.InLinks(*po.link_rows(src, dst, n), n)


def _pr_step(L, n, x, addend, xoff=0, yoff=0):
    """One mb_pagerank_step; x inside a NaN parent at xoff, y inside a sentinel parent at yoff.  Returns (y, untouched)."""
    import torch
    import marlin_b200 as mb
    rt = mb.Runtime.get()
    xh = np.full(xoff + n + 2, np.nan)
    xh[xoff: xoff + n] = x
    yh = np.full(yoff + n + 2, SENTINEL)
    xt, yt = torch.from_numpy(xh).cuda(), torch.from_numpy(yh).cuda()
    xv = mb.SubMatrix(buf=xt, rows=n, cols=1, ld=n, offset=xoff)
    yv = mb.SubMatrix(buf=yt, rows=n, cols=1, ld=n, offset=yoff)
    rt.sync_stream()
    nat.check(rt.lib.mb_pagerank_step(rt.ctx, L.handle(), xv.handle(), (n + 1) // 2, addend, yv.handle()))
    rt.synchronize()
    out = yt.cpu().numpy()
    return out[yoff: yoff + n].copy(), _outside_untouched(yt, yoff, n, 1, n, False)


def test_pagerank_step_power_of_two_scaling(pr_graph):
    """x -> 2^k x with addend -> 2^k addend gives y -> 2^k y: the link weights are fixed and every term is w x_j.  With
    x in [0.5, 1) and weights >= 2^-14 every nonzero term and partial sum lies in [2^-15, 2^13], so |k| <= 500 keeps them
    normal.  The unscaled step is the oracle's bit for bit."""
    n, _, _, L, oracle = pr_graph
    x = 0.5 + 0.5 * np.random.default_rng(4).random(n)
    base, _ = _pr_step(L, n, x, 0.15)
    assert identical(base, oracle.step(x, 0.15))
    for k in (1, -1, 37, -37, 500, -500):
        assert identical(_pr_step(L, n, x * p2(k), 0.15 * p2(k))[0], np.ldexp(base, k)), k


def test_pagerank_step_views_in_poisoned_parents(pr_graph):
    n, _, _, L, _ = pr_graph
    x = np.random.default_rng(5).random(n)
    want, _ = _pr_step(L, n, x, 0.15)
    for xoff, yoff in [(1, 3), (2, 1), (3, 2)]:
        got, untouched = _pr_step(L, n, x, 0.15, xoff, yoff)
        assert untouched and identical(got, want), (xoff, yoff)


@pytest.mark.parametrize("poison", [np.nan, np.inf])
def test_pagerank_nan_or_inf_rank_reaches_exactly_the_pages_it_links_to(pr_graph, poison):
    """x_p poisoned for pages in both segments, with light and heavy targets among their out-links: y_i is NaN (or +Inf:
    every weight is positive) exactly for the pages i that p links to, and every other y_i keeps its bits."""
    n, src, dst, L, _ = pr_graph
    x = np.random.default_rng(6).random(n)
    clean, _ = _pr_step(L, n, x, 0.15)
    outs = np.bincount(src, minlength=n)
    pages = [int(np.argmax(outs[: n // 2])), int(n // 2 + np.argmax(outs[n // 2:])), int(np.flatnonzero(outs == outs[outs > 0].min())[0])]
    xp = x.copy()
    xp[pages] = poison
    got, _ = _pr_step(L, n, xp, 0.15, 1, 1)
    hit = np.zeros(n, bool)
    hit[dst[np.isin(src, pages)]] = True
    assert hit.any() and (np.all(np.isnan(got[hit])) if np.isnan(poison) else np.all(np.isposinf(got[hit])))
    assert identical(got[~hit], clean[~hit])

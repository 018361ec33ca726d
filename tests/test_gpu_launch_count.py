"""mb_launch_count: the kernels the calls on a context have enqueued.  Each launch site in marlin_b200/csrc counts itself
through one helper (csrc/launch.h), so the count is exact per call:
  * non-empty inputs: the per-entry counts pinned below (the factorizations through a model of their recursion);
  * a call that launches nothing (an empty block, an empty side, nnz = 0) adds nothing."""
import ctypes as C
import re
from pathlib import Path

import numpy as np
import pytest

from marlin_b200 import _native as nat

CSRC = Path(__file__).resolve().parents[1] / "marlin_b200" / "csrc"


def _sources():
    return [(p, p.read_text()) for p in sorted(CSRC.iterdir()) if p.is_file()]


def test_launches_are_counted_only_by_the_launch_helper():
    params = [f"{p.name}: {m.group(0)}" for p, text in _sources() for m in re.finditer(r"\*\s*launches\b", text)]
    assert params == [], "launchers take no launch-count parameter: a launch counts itself with mb::launched()"
    adds = [f"{p.name}:{i}" for p, text in _sources() if p.name != "launch.h"
            for i, line in enumerate(text.splitlines(), 1)
            if re.search(r"launches\s*(\+\+|\+=|-=|=[^=]|\.\s*fetch_add|\.\s*store)|\+\+\s*\*?\s*(\w+->)?launches", line)]
    assert adds == [], "only csrc/launch.h adds to a launch count"
    assert not any("flag_wait_bounded" in text for _, text in _sources())


# ---------------------------------------------------------------------------------------------------------------- GPU
def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class _Env:
    def __init__(self):
        import marlin_b200 as mb
        self.rt = mb.Runtime.get()
        self.lib, self.ctx = self.rt.lib, self.rt.ctx
        self.blocks, self.sparse, self.keep = [], [], []

    def count(self, call):
        """Launches one successful call adds to the context's count."""
        l0 = self.lib.mb_launch_count(self.ctx)
        rc = call()
        assert rc == nat.MB_OK, self.lib.mb_last_error()
        nat.check(self.lib.mb_synchronize(self.ctx))
        return self.lib.mb_launch_count(self.ctx) - l0

    def block(self, a):
        f = np.asfortranarray(np.asarray(a, np.float64).reshape(np.shape(a)))
        self.keep.append(f)
        h = nat.c_blk()
        nat.check(self.lib.mb_block_upload(self.ctx, _p(f) if f.size else _p(np.zeros(1)), 0, f.shape[0], f.shape[1],
                                           max(1, f.shape[0]), 0, nat.MB_F64, C.byref(h)))
        self.blocks.append(h)
        return h

    def empty(self, rows, cols):
        h = nat.c_blk()
        nat.check(self.lib.mb_block_alloc(self.ctx, rows, cols, nat.MB_F64, C.byref(h)))
        self.blocks.append(h)
        return h

    def rows(self, X):
        """A row-major view of X, as ALS and logistic regression read rows."""
        v = nat.c_blk()
        nat.check(self.lib.mb_block_view_t(self.ctx, self.block(np.asarray(X, np.float64).T), C.byref(v)))
        self.blocks.append(v)
        return v

    def csc(self, rows, cols, colptr, rowidx, values):
        arrs = (np.ascontiguousarray(colptr, np.int32), np.ascontiguousarray(rowidx, np.int32),
                np.ascontiguousarray(values, np.float64))
        self.keep.extend(arrs)
        s = nat.c_sp()
        nat.check(self.lib.mb_sparse_upload(self.ctx, rows, cols, *[_p(a) if a.size else _p(np.zeros(1)) for a in arrs],
                                            C.byref(s)))
        self.sparse.append(s)
        return s

    def close(self):
        for s in self.sparse:
            self.lib.mb_sparse_free(self.ctx, s)
        for h in reversed(self.blocks):
            self.lib.mb_block_free(self.ctx, h)


@pytest.fixture(scope="module")
def env():
    e = _Env()
    yield e
    e.close()


# The recursion of csrc/factor.cu, one count per kernel or GEMM launch.
LEAF, PANEL_W = 64, 32


def _split(n):
    h = (n // 2 + 31) // 32 * 32
    if h >= n:
        h = n // 2 // 32 * 32
    return h if h > 0 else n // 2


def _trsm(t, nrhs):
    if t <= 0 or nrhs <= 0:
        return 0
    if t <= LEAF:
        return 1
    h = _split(t)
    return _trsm(h, nrhs) + 1 + _trsm(t - h, nrhs)


def _getrf(m, n):
    if m <= 0 or n <= 0:
        return 0
    if n <= PANEL_W:
        return 1
    n1 = min(_split(n), m)
    k1 = min(m, n1)
    c = _getrf(m, n1) + 1 + _trsm(k1, n - n1)              # left half, its interchanges on the right, U12
    if m > k1:
        c += 1 + _getrf(m - k1, n - n1) + 1                 # A22 update, right half, its interchanges on the left
    return c


def _potrf(n):
    if n <= 0:
        return 0
    if n <= LEAF:
        return 1
    n1 = _split(n)
    return _potrf(n1) + _trsm(n1, n - n1) + 1 + _potrf(n - n1)


@pytest.mark.gpu
def test_elementwise_and_vector_entries(env):
    lib, ctx = env.lib, env.ctx
    rng = np.random.default_rng(0)
    A, B, out = env.block(rng.standard_normal((300, 200))), env.block(rng.standard_normal((300, 200))), env.empty(300, 200)
    outT = env.empty(200, 300)
    assert env.count(lambda: lib.mb_block_add(ctx, A, B, out)) == 1
    assert env.count(lambda: lib.mb_block_axpb(ctx, A, 2.0, 1.0, out)) == 1
    assert env.count(lambda: lib.mb_block_copy(ctx, A, out)) == 1
    assert env.count(lambda: lib.mb_block_transpose(ctx, A, outT)) == 1
    s = C.c_double()
    assert env.count(lambda: lib.mb_block_sum(ctx, A, C.byref(s))) == 2
    x, y = env.block(rng.standard_normal((200, 1))), env.empty(300, 1)
    assert env.count(lambda: lib.mb_block_dot(ctx, x, x, C.byref(s))) == 2
    assert env.count(lambda: lib.mb_block_gemv(ctx, A, x, y, 0)) == 2
    At = nat.c_blk()
    nat.check(lib.mb_block_view_t(ctx, A, C.byref(At)))
    env.blocks.append(At)
    assert env.count(lambda: lib.mb_block_gemv(ctx, At, y, x, 1)) == 2
    yr = env.block(rng.standard_normal((1, 200)))
    assert env.count(lambda: lib.mb_block_ger(ctx, y, yr, out)) == 1


@pytest.mark.gpu
def test_factorization_entries(env):
    lib, ctx = env.lib, env.ctx
    rng = np.random.default_rng(1)
    m, n = 300, 200
    assert env.count(lambda: lib.mb_block_lu(ctx, env.block(rng.standard_normal((m, n))), None)) == _getrf(m, n)
    X = rng.standard_normal((n, n))
    assert env.count(lambda: lib.mb_block_cholesky(ctx, env.block(X @ X.T + n * np.eye(n)))) == _potrf(n) + 1
    k = 150
    inv = env.empty(k, k)
    # the working copy, the LU, the permuted identity (2), two triangular solves
    assert env.count(lambda: lib.mb_block_inverse(ctx, env.block(rng.standard_normal((k, k)) + k * np.eye(k)), inv)) == \
        1 + _getrf(k, k) + 2 + 2 * _trsm(k, k)
    T = env.block(np.tril(rng.standard_normal((n, n))) + n * np.eye(n))
    assert env.count(lambda: lib.mb_block_trsm(ctx, T, 1, 0, env.block(rng.standard_normal((n, 50))))) == _trsm(n, 50)


@pytest.mark.gpu
def test_svd_and_lr_entries(env):
    lib, ctx = env.lib, env.ctx
    rng = np.random.default_rng(2)
    G = env.empty(96, 96)
    assert env.count(lambda: lib.mb_block_gramian(ctx, env.block(rng.standard_normal((1000, 96))), G)) == 2
    n = 37
    S = rng.standard_normal((n, n))
    V, w, sweeps = env.empty(n, n), np.empty(n), C.c_int32()
    got = env.count(lambda: lib.mb_block_syev(ctx, env.block(S + S.T), V, w.ctypes.data_as(nat.c_dp), C.byref(sweeps)))
    assert sweeps.value > 0 and got == 3 + sweeps.value * 37       # padded to N = 38: a sweep is N - 1 rounds
    X = env.rows(np.column_stack([rng.integers(0, 2, 500), rng.standard_normal((500, 9))]))
    wv, g = np.zeros(10), np.empty(10)
    assert env.count(lambda: lib.mb_lr_gradient(ctx, X, wv.ctypes.data_as(nat.c_dp), g.ctypes.data_as(nat.c_dp))) == 2
    assert env.count(lambda: lib.mb_lr_train(ctx, X, 500, 1.0, 3, g.ctypes.data_as(nat.c_dp))) == 2 * 3


def _als(env, seed=3, rank=4, work=None):
    import torch
    from marlin_b200.matrix.coordinate_matrix import _Links
    rng = np.random.default_rng(seed)
    r, c = rng.integers(0, 40, 400), rng.integers(0, 30, 400)
    users, products = _Links(r, c, rng.integers(1, 6, 400).astype(np.float32), 2, 2), _Links(c, r, np.ones(400, np.float32), 2, 2)
    side, keep = users.to_device(env.rt.device, work)
    torch.cuda.synchronize()
    env.keep.append(keep)
    return side, env.rows(rng.random((products.n, rank))), env.rows(np.zeros((users.n, rank)))


@pytest.mark.gpu
def test_als_and_coo_entries(env):
    lib, ctx = env.lib, env.ctx
    side, Y, X = _als(env)
    assert env.count(lambda: lib.mb_als_update(ctx, C.byref(side), Y, 0.1, 1.0, 0, None, X)) == 1
    out = env.rows(np.zeros((6, 5)))
    rp, cp, vp = np.array([0, 5, 2], np.int32), np.array([4, 0, 3], np.int32), np.array([1.5, -2.0, 3.0], np.float32)
    assert env.count(lambda: lib.mb_coo_to_dense_rows(ctx, 3, _p(rp), _p(cp), _p(vp), out)) == 1


def _links(env, n, sources_of):
    """In-links of n pages as the PageRank entries read them: the CSC of the transpose, one column per target."""
    ptr = np.concatenate([[0], np.cumsum([len(s) for s in sources_of])])
    idx = np.concatenate([sorted(s) for s in sources_of])
    return env.csc(n, n, ptr, idx, np.full(idx.size, 0.5))


@pytest.mark.gpu
def test_sparse_and_pagerank_entries(env):
    import scipy.sparse
    lib, ctx = env.lib, env.ctx
    rng = np.random.default_rng(4)
    S = scipy.sparse.random(50, 40, density=0.2, format="csc", random_state=5)
    S.sort_indices()
    A = env.csc(50, 40, S.indptr, S.indices, S.data)
    assert env.count(lambda: lib.mb_sparse_to_dense(ctx, A, env.empty(50, 40))) == 1
    assert env.count(lambda: lib.mb_spmm_dense_sparse(ctx, env.block(rng.standard_normal((30, 50))), A, env.empty(30, 40), 0)) == 1
    Bd, Cd = env.block(rng.standard_normal((40, 30))), env.empty(50, 30)
    assert env.count(lambda: lib.mb_spmm_sparse_dense(ctx, A, Bd, Cd, 0)) == 4 + 1       # the CSR copy on first use
    assert env.count(lambda: lib.mb_spmm_sparse_dense(ctx, A, Bd, Cd, 1)) == 1
    T = scipy.sparse.random(40, 20, density=0.3, format="csc", random_state=6)
    T.sort_indices()
    assert env.count(lambda: lib.mb_spgemm_dense_out(ctx, A, env.csc(40, 20, T.indptr, T.indices, T.data), env.empty(50, 20), 0)) == 1
    R = nat.c_sp()
    nat.check(lib.mb_sparse_alloc(ctx, 50, 20, 20 * 5, C.byref(R)))
    env.sparse.append(R)
    assert env.count(lambda: lib.mb_fill_sparse_uniform(ctx, R, 11)) == 2               # values (general kernel), rows

    n = 600
    L = _links(env, n, [list(range(n))] + [[i - 1] for i in range(1, n)])              # page 0 has n > 256 in-links
    x, y = env.block(np.full((n, 1), 1.0 / n)), env.empty(n, 1)
    assert env.count(lambda: lib.mb_pagerank_step(ctx, L, x, 1 << 20, 0.15, y)) == 1 + 2   # binning, light and heavy rows
    assert env.count(lambda: lib.mb_pagerank_step(ctx, L, x, 1 << 20, 0.15, y)) == 2


@pytest.mark.gpu
def test_calls_that_launch_nothing_count_nothing(env):
    lib, ctx = env.lib, env.ctx
    E, F, G = env.empty(0, 5), env.empty(0, 5), env.empty(5, 0)
    for name, call in {
        "add": lambda: lib.mb_block_add(ctx, E, F, E),
        "sub": lambda: lib.mb_block_sub(ctx, E, F, E),
        "hadamard": lambda: lib.mb_block_hadamard(ctx, E, F, E),
        "axpb": lambda: lib.mb_block_axpb(ctx, E, 2.0, 1.0, F),
        "fill": lambda: lib.mb_block_fill(ctx, E, 3.0),
        "div": lambda: lib.mb_block_div(ctx, E, 2.0, 1, F),
        "copy": lambda: lib.mb_block_copy(ctx, E, F),
        "transpose": lambda: lib.mb_block_transpose(ctx, E, G),
        "ger": lambda: lib.mb_block_ger(ctx, env.empty(0, 1), env.empty(1, 5), E),
    }.items():
        assert env.count(call) == 0, name

    S0 = env.csc(0, 4, np.zeros(5), [], [])                                           # no rows
    A = env.csc(4, 3, [0, 1, 2, 3], [0, 1, 2], [1.0, 2.0, 3.0])
    assert env.count(lambda: lib.mb_sparse_to_dense(ctx, S0, env.empty(0, 4))) == 0
    assert env.count(lambda: lib.mb_spmm_dense_sparse(ctx, env.empty(0, 4), A, env.empty(0, 3), 0)) == 0
    assert env.count(lambda: lib.mb_spmm_sparse_dense(ctx, S0, env.empty(4, 3), env.empty(0, 3), 0)) == 0
    assert env.count(lambda: lib.mb_spgemm_dense_out(ctx, S0, A, env.empty(0, 3), 0)) == 0

    side, Y, X = _als(env, work=np.empty(0, np.int32))                                # a side with no entities
    assert side.count == 0
    assert env.count(lambda: lib.mb_als_update(ctx, C.byref(side), Y, 0.1, 1.0, 0, None, X)) == 0
    none = np.zeros(1, np.int32)
    assert env.count(lambda: lib.mb_coo_to_dense_rows(ctx, 0, _p(none), _p(none), _p(none), env.rows(np.ones((3, 2))))) == 0

    n = 100                                                                          # too few links for a heavy row
    L = _links(env, n, [[(i - 1) % n, (i + 1) % n] for i in range(n)])
    x, y = env.block(np.full((n, 1), 1.0 / n)), env.empty(n, 1)
    assert env.count(lambda: lib.mb_pagerank_step(ctx, L, x, 1 << 20, 0.15, y)) == 1     # light rows only, no binning kernel

"""Per-call device temporaries of the C ABI.  Every one comes from one stream-ordered owner (marlin_b200/csrc/stream_buffer.h):
each entry below takes memory from the device's default pool and has returned all of it once its stream is synchronised,
also when it fails after taking it.  A handle-creating entry that fails sets *out to NULL.

The pool counters are read through the driver API (CU_MEMPOOL_ATTR_USED_MEM_*): they count this process's allocations
only, so other work on the same GPU does not move them."""
import ctypes as C
import re
from pathlib import Path

import numpy as np
import pytest

from marlin_b200 import _native as nat

ROOT = Path(__file__).resolve().parents[1]
CSRC = ROOT / "marlin_b200" / "csrc"
CU_MEMPOOL_ATTR_USED_MEM_CURRENT, CU_MEMPOOL_ATTR_USED_MEM_HIGH = 7, 8


def test_stream_ordered_allocation_only_in_the_owner():
    hits = [f"{p.name}:{i}" for p in sorted(CSRC.iterdir()) if p.is_file() and p.name != "stream_buffer.h"
            for i, line in enumerate(p.read_text().splitlines(), 1) if re.search(r"cudaMallocAsync|cudaFreeAsync", line)]
    assert hits == [], "per-call device memory belongs in mb::StreamBuffer"


class _Pool:
    """The default memory pool of CUDA device 0 (the Runtime's device in a single-process run)."""

    def __init__(self):
        cu = C.CDLL("libcuda.so.1")
        cu.cuDeviceGetDefaultMemPool.argtypes = [C.POINTER(C.c_void_p), C.c_int]
        cu.cuMemPoolGetAttribute.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        cu.cuMemPoolSetAttribute.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        assert cu.cuInit(0) == 0
        self.cu, self.pool = cu, C.c_void_p()
        assert cu.cuDeviceGetDefaultMemPool(C.byref(self.pool), 0) == 0

    def _attr(self, attr):
        v = C.c_uint64()
        assert self.cu.cuMemPoolGetAttribute(self.pool, attr, C.byref(v)) == 0
        return v.value

    def used(self):
        return self._attr(CU_MEMPOOL_ATTR_USED_MEM_CURRENT)

    def reset_high(self):
        zero = C.c_uint64(0)
        assert self.cu.cuMemPoolSetAttribute(self.pool, CU_MEMPOOL_ATTR_USED_MEM_HIGH, C.byref(zero)) == 0

    def high(self):
        return self._attr(CU_MEMPOOL_ATTR_USED_MEM_HIGH)


class _Env:
    def __init__(self):
        import marlin_b200 as mb
        self.rt = mb.Runtime.get()
        self.rt.sync_stream()
        self.lib, self.ctx = self.rt.lib, self.rt.ctx
        self.pool = _Pool()
        self.blocks, self.sparse, self.keep = [], [], []

    def block(self, a, dtype=nat.MB_F64):
        f = np.asfortranarray(a, np.float64)
        self.keep.append(f)
        h = nat.c_blk()
        nat.check(self.lib.mb_block_upload(self.ctx, _p(f), 0, f.shape[0], f.shape[1], max(1, f.shape[0]), 0, dtype, C.byref(h)))
        self.blocks.append(h)
        return h

    def rows(self, X):
        """A row-major view of X (one row per matrix row), as ALS and PageRank read factors and rows."""
        v = nat.c_blk()
        nat.check(self.lib.mb_block_view_t(self.ctx, self.block(np.asarray(X, np.float64).T), C.byref(v)))
        self.blocks.append(v)
        return v

    def csc(self, rows, cols, colptr, rowidx, values):
        arrs = (np.ascontiguousarray(colptr, np.int32), np.ascontiguousarray(rowidx, np.int32),
                np.ascontiguousarray(values, np.float64))
        self.keep.extend(arrs)
        s = nat.c_sp()
        nat.check(self.lib.mb_sparse_upload(self.ctx, rows, cols, *map(_p, arrs), C.byref(s)))
        self.sparse.append(s)
        return s

    def balanced(self, call, expect=nat.MB_OK):
        """Warm the entry, then check that the second call takes pool memory and has returned it after a synchronise."""
        assert call() == expect, self.lib.mb_last_error()
        nat.check(self.lib.mb_synchronize(self.ctx))
        before = self.pool.used()
        self.pool.reset_high()
        assert call() == expect, self.lib.mb_last_error()
        nat.check(self.lib.mb_synchronize(self.ctx))
        assert self.pool.high() > before, "the call took no temporary from the pool"
        assert self.pool.used() == before

    def close(self):
        for s in self.sparse:
            self.lib.mb_sparse_free(self.ctx, s)
        for h in reversed(self.blocks):
            self.lib.mb_block_free(self.ctx, h)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def env():
    e = _Env()
    yield e
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("store, trans", [(nat.MB_BF16, 0), (nat.MB_F64, 1), (nat.MB_BF16, 1)])
def test_upload_and_download_stage_through_the_pool(env, store, trans):
    rng = np.random.default_rng(0)
    host = rng.standard_normal(301 * 203)
    out = np.empty((203, 301) if trans else (301, 203), order="F")
    blk = nat.c_blk()

    def upload():
        rc = env.lib.mb_block_upload(env.ctx, _p(host), 0, out.shape[0], out.shape[1], 301, trans, store, C.byref(blk))
        if rc == nat.MB_OK:
            env.lib.mb_block_free(env.ctx, blk)
        return rc

    env.balanced(upload)
    src = env.block(rng.standard_normal((97, 61)), store)
    view = nat.c_blk()
    nat.check(env.lib.mb_block_view_t(env.ctx, src, C.byref(view)))
    env.blocks.append(view)
    shape = (61, 97) if trans else (97, 61)
    dst = np.empty(shape, order="F")
    env.balanced(lambda: env.lib.mb_block_download(env.ctx, view if trans else src, _p(dst), shape[0]))


@pytest.mark.gpu
def test_dgemm_host(env):
    rng = np.random.default_rng(1)
    m, n, k = 67, 45, 33
    a, b = np.asfortranarray(rng.standard_normal((m, k))), np.asfortranarray(rng.standard_normal((n, k)))
    c = np.asfortranarray(rng.standard_normal((m, n)))
    env.balanced(lambda: env.lib.mb_dgemm_host(env.ctx, b"N", b"T", m, n, k, 1.0, _p(a), 0, m, _p(b), 0, n, 0.5, _p(c), 0, m))


@pytest.mark.gpu
def test_bf16_gemm_stages_odd_leading_dimensions(env):
    rng = np.random.default_rng(2)
    A, B = env.block(rng.standard_normal((37, 64)), nat.MB_BF16), env.block(rng.standard_normal((64, 40)), nat.MB_BF16)
    Cb = nat.c_blk()
    nat.check(env.lib.mb_block_alloc(env.ctx, 37, 40, nat.MB_F32, C.byref(Cb)))
    env.blocks.append(Cb)
    env.balanced(lambda: env.lib.mb_block_gemm(env.ctx, A, B, Cb, 0))        # A's ld is 37: it is staged


@pytest.mark.gpu
def test_gramian_split_k(env):
    import torch
    m, n = 1 << 16, 128
    assert env.lib.mb_gramian_workspace_bytes(n, m, torch.cuda.get_device_properties(0).multi_processor_count) > 0
    A, G = nat.c_blk(), nat.c_blk()
    nat.check(env.lib.mb_block_alloc(env.ctx, m, n, nat.MB_F64, C.byref(A)))
    nat.check(env.lib.mb_block_alloc(env.ctx, n, n, nat.MB_F64, C.byref(G)))
    env.blocks += [A, G]
    nat.check(env.lib.mb_fill_uniform(env.ctx, A, 7, 0, -1.0, 1.0, 0))
    env.balanced(lambda: env.lib.mb_block_gramian(env.ctx, A, G))


@pytest.mark.gpu
def test_lr_on_a_column_major_block(env):
    rng = np.random.default_rng(3)
    X = env.block(np.column_stack([rng.integers(0, 2, 500), rng.standard_normal((500, 9))]))
    w, g = np.zeros(10), np.empty(10)
    env.balanced(lambda: env.lib.mb_lr_gradient(env.ctx, X, w.ctypes.data_as(nat.c_dp), g.ctypes.data_as(nat.c_dp)))
    env.balanced(lambda: env.lib.mb_lr_train(env.ctx, X, 500, 1.0, 3, g.ctypes.data_as(nat.c_dp)))


def _als_case(seed, rank=4):
    from marlin_b200.matrix.coordinate_matrix import _Links
    rng = np.random.default_rng(seed)
    rows, cols = rng.integers(0, 40, 400), rng.integers(0, 30, 400)
    vals = rng.integers(1, 6, 400).astype(np.float32)
    return _Links(rows, cols, vals, 2, 2), _Links(cols, rows, vals, 2, 2), rank


@pytest.mark.gpu
def test_als(env):
    import torch
    users, products, rank = _als_case(4)
    side, keep = users.to_device(env.rt.device)
    torch.cuda.synchronize()
    rng = np.random.default_rng(5)
    Y, X = env.rows(rng.random((products.n, rank))), env.rows(np.zeros((users.n, rank)))
    env.balanced(lambda: env.lib.mb_als_update(env.ctx, C.byref(side), Y, 0.1, 1.0, 1, None, X))     # implicit, YtY computed

    Yh, Xh = rng.random((products.n, rank)), np.zeros((users.n, rank))
    env.balanced(lambda: env.lib.mb_als_update_host(env.ctx, rank, products.n, _p(Yh), users.n, _p(users.ids), _p(users.offsets),
                                                    _p(users.partners), _p(users.ratings), 0.1, 1.0, 1, None, _p(Xh)))

    out = env.rows(np.zeros((6, 5)))
    rp, cp, vp = np.array([0, 5, 2], np.int32), np.array([4, 0, 3], np.int32), np.array([1.5, -2.0, 3.0], np.float32)
    env.balanced(lambda: env.lib.mb_coo_to_dense_rows(env.ctx, 3, _p(rp), _p(cp), _p(vp), out))
    del keep


@pytest.mark.gpu
def test_spvec_multiply_in_all_three_bins_and_dense_rows(env):
    rng = np.random.default_rng(6)
    n, K = 40000, 100
    b_ptr = np.arange(K + 1) * 64
    b_idx = np.concatenate([np.sort(rng.choice(n, 64, replace=False)) for _ in range(K)])
    B = env.csc(n, K, b_ptr, b_idx, rng.standard_normal(b_idx.size))                  # K rows of n columns
    counts = [2, 10, K]                          # 128, 640 and 6400 products: warp, CTA and window bins
    assert counts[0] * 64 <= nat.MB_SPVEC_WARP_BOUND < counts[1] * 64 <= nat.MB_SPVEC_CTA_BOUND < counts[2] * 64
    a_ptr = np.concatenate([[0], np.cumsum(counts)])
    a_idx = np.concatenate([np.sort(rng.choice(K, c, replace=False)) for c in counts])
    A = env.csc(K, len(counts), a_ptr, a_idx, rng.standard_normal(a_idx.size))
    out = nat.c_sp()

    def multiply():
        l0 = env.lib.mb_launch_count(env.ctx)
        rc = env.lib.mb_spvec_multiply(env.ctx, A, B, C.byref(out))
        if rc == nat.MB_OK:
            assert env.lib.mb_launch_count(env.ctx) - l0 == 8             # bound, 3 count bins, scan, 3 fill bins
            env.lib.mb_sparse_free(env.ctx, out)
        return rc

    env.balanced(multiply)
    D = env.rows(rng.standard_normal((50, 30)) * (rng.random((50, 30)) < 0.3))

    def to_sparse():
        rc = env.lib.mb_dense_rows_to_sparse(env.ctx, D, C.byref(out))
        if rc == nat.MB_OK:
            env.lib.mb_sparse_free(env.ctx, out)
        return rc

    env.balanced(to_sparse)


@pytest.mark.gpu
def test_spmm_sparse_dense_csr_copy(env):
    import scipy.sparse
    rng = np.random.default_rng(7)
    S = scipy.sparse.random(50, 40, density=0.2, format="csc", random_state=8)
    S.sort_indices()
    Bd, Cd = env.block(rng.standard_normal((40, 30))), env.block(np.zeros((50, 30)))
    arrs = (S.indptr.astype(np.int32), S.indices.astype(np.int32), S.data.astype(np.float64))
    fresh = nat.c_sp()

    def spmm():                                  # a fresh handle each time: the CSR copy is built on its first product
        nat.check(env.lib.mb_sparse_upload(env.ctx, 50, 40, *map(_p, arrs), C.byref(fresh)))
        rc = env.lib.mb_spmm_sparse_dense(env.ctx, fresh, Bd, Cd, 0)
        env.lib.mb_sparse_free(env.ctx, fresh)
        return rc

    env.balanced(spmm)


@pytest.mark.gpu
def test_pagerank_train(env):
    n = 1000
    colptr = np.arange(n + 1) * 2
    rowidx = np.array([sorted(((i - 1) % n, (i + 1) % n)) for i in range(n)]).reshape(-1)
    L = env.csc(n, n, colptr, rowidx, np.full(2 * n, 0.425))
    x = env.block(np.ones((n, 1)))
    env.balanced(lambda: env.lib.mb_pagerank_train(env.ctx, L, n, 0.15, 3, x))


@pytest.mark.gpu
def test_failures_after_taking_memory_return_it(env):
    A, out = env.block(np.zeros((8, 8))), env.block(np.zeros((8, 8)))
    env.balanced(lambda: env.lib.mb_block_inverse(env.ctx, A, out), nat.MB_ERR_CUDA)
    assert b"singular" in env.lib.mb_last_error()

    import torch
    users, products, rank = _als_case(9)
    side, keep = users.to_device(env.rt.device)
    torch.cuda.synchronize()
    Y, X = env.rows(np.zeros((products.n, rank))), env.rows(np.zeros((users.n, rank)))
    # implicit, YtY computed from Y = 0 and lambda = 0: every A_u is zero, so the Cholesky pivot check fails
    env.balanced(lambda: env.lib.mb_als_update(env.ctx, C.byref(side), Y, 0.0, 1.0, 1, None, X), nat.MB_ERR_CUDA)
    assert b"not positive definite" in env.lib.mb_last_error()
    del keep


@pytest.mark.gpu
def test_failing_handle_entries_leave_out_null(env):
    lib, ctx = env.lib, env.ctx
    blk = env.block(np.ones((4, 4)))
    bf16 = env.block(np.ones((4, 4)), nat.MB_BF16)
    host = np.ones(16)
    dev = C.c_void_p()
    nat.check(lib.mb_block_info(blk, None, None, None, None, None, C.byref(dev)))
    bad_colptr = np.array([0, 2, 1], np.int32)
    idx, val = np.array([0, 1], np.int32), np.array([1.0, 2.0])
    S = env.csc(2, 2, [0, 1, 2], [0, 1], [1.0, 2.0])
    S3 = env.csc(3, 2, [0, 1, 2], [0, 2], [1.0, 2.0])
    entries = {
        "mb_block_alloc": lambda o: lib.mb_block_alloc(ctx, 2, 2, 7, o),                                  # bad dtype
        "mb_block_wrap": lambda o: lib.mb_block_wrap(ctx, dev, 0, 4, 4, 2, 0, nat.MB_F64, o),              # bad ld
        "mb_block_upload": lambda o: lib.mb_block_upload(ctx, _p(host), 0, 4, 4, 2, 0, nat.MB_F64, o),     # bad ld
        "mb_block_view_t": lambda o: lib.mb_block_view_t(ctx, None, o),                                    # no block
        "mb_block_slice": lambda o: lib.mb_block_slice(ctx, blk, 0, 5, 0, 1, o),                           # bad range
        "mb_sparse_wrap": lambda o: lib.mb_sparse_wrap(ctx, 2, 2, -1, dev, dev, dev, o),                   # bad nnz
        "mb_sparse_upload": lambda o: lib.mb_sparse_upload(ctx, 2, 2, _p(bad_colptr), _p(idx), _p(val), o),  # bad colptr
        "mb_sparse_alloc": lambda o: lib.mb_sparse_alloc(ctx, 2, 2, -1, o),                                # bad nnz
        "mb_sparse_values_op": lambda o: lib.mb_sparse_values_op(ctx, S, 9, 1.0, o),                       # bad op
        "mb_spvec_multiply": lambda o: lib.mb_spvec_multiply(ctx, S3, S, o),                               # dimension mismatch
        "mb_spvec_multiply_host": lambda o: lib.mb_spvec_multiply_host(ctx, 2, 2, _p(bad_colptr), _p(idx), _p(val), 2,
                                                                       _p(bad_colptr), _p(idx), _p(val), o),  # bad colptr
        "mb_dense_rows_to_sparse": lambda o: lib.mb_dense_rows_to_sparse(ctx, bf16, o),                    # bad dtype
    }
    for name, call in entries.items():
        out = C.c_void_p(0x5E47)
        assert call(C.byref(out)) != nat.MB_OK, name
        assert out.value is None, f"{name} left *out set after failing"

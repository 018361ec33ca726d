"""Sparse blocks on the H100: the LocalMatrixSuite cases, bit-identity of toDense and the three products with the host
restatement of the reference loops (tests/sparse_oracle.py), accumulate, the scalar ops, the generator, and
BlockMatrix.multiply / multiply(BDM) / multiplyBy with sparse blocks."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import marlin_b200 as mb
from marlin_b200 import _native as nat
from marlin_b200.matrix.sparse_matrix import SparseBlock, SparseMatrix, SparseVector
from marlin_b200.utils.mt_utils import MTUtils, UniformGenerator

from tests import sparse_oracle as so
from tests.test_oracle_sparse import (DENSE, EXPECTED_DENSE_SPARSE, EXPECTED_SPARSE_DENSE, EXPECTED_SPARSE_SPARSE,
                                      EXPECTED_TO_DENSE, suite_csc, suite_matrix)


def sp(S) -> mb.SubMatrix:
    return mb.SubMatrix(sparse=SparseBlock.from_host(*S))


def same(a, b) -> bool:
    """Bitwise equality (so -0.0 != 0.0), except that any NaN equals any NaN: host and device may pick different NaN
    payloads."""
    a, b = np.ascontiguousarray(a, dtype=np.float64), np.ascontiguousarray(b, dtype=np.float64)
    if a.shape != b.shape or not np.array_equal(np.isnan(a), np.isnan(b)):
        return False
    keep = ~np.isnan(a)
    return np.array_equal(a[keep].view(np.int64), b[keep].view(np.int64))


def test_local_matrix_suite_through_the_c_abi():
    rt = mb.Runtime.get()
    lib = rt.lib
    cp, ri, va = suite_matrix().to_csc()
    S = nat.c_sp()
    nat.check(lib.mb_sparse_upload(rt.ctx, 4, 4, cp.ctypes.data, ri.ctypes.data, va.ctypes.data, C.byref(S)))
    try:
        rows, cols, nnz = C.c_int32(), C.c_int32(), C.c_int64()
        nat.check(lib.mb_sparse_info(S, C.byref(rows), C.byref(cols), C.byref(nnz)))
        assert (rows.value, cols.value, nnz.value) == (4, 4, 5)
        back = (np.zeros(5, np.int32), np.zeros(5, np.int32), np.zeros(5))
        nat.check(lib.mb_sparse_download(rt.ctx, S, back[0].ctypes.data, back[1].ctypes.data, back[2].ctypes.data))
        assert np.array_equal(back[0], cp) and np.array_equal(back[1], ri) and np.array_equal(back[2], va)
        D = mb.SubMatrix(DENSE)
        outs = [mb.SubMatrix.zeros(4, 4) for _ in range(4)]
        nat.check(lib.mb_sparse_to_dense(rt.ctx, S, outs[0].handle()))
        nat.check(lib.mb_spmm_dense_sparse(rt.ctx, D.handle(), S, outs[1].handle(), 0))
        nat.check(lib.mb_spgemm_dense_out(rt.ctx, S, S, outs[2].handle(), 0))
        nat.check(lib.mb_spmm_sparse_dense(rt.ctx, S, D.handle(), outs[3].handle(), 0))
        for o, e in zip(outs, [EXPECTED_TO_DENSE, EXPECTED_DENSE_SPARSE, EXPECTED_SPARSE_SPARSE, EXPECTED_SPARSE_DENSE]):
            assert same(o.toBreeze(), e)
        bad = np.array([0, 2], np.int32), np.array([1, 1], np.int32)
        with pytest.raises(nat.MarlinArgumentError, match="not strictly increasing"):
            nat.check(lib.mb_sparse_upload(rt.ctx, 4, 1, bad[0].ctypes.data, bad[1].ctypes.data, va.ctypes.data,
                                           C.byref(nat.c_sp())))
    finally:
        lib.mb_sparse_free(rt.ctx, S)


def test_local_matrix_suite_through_submatrix():
    S = mb.SubMatrix(spMatrix=suite_matrix())
    D = mb.SubMatrix(DENSE)
    assert S.isSparse and not D.isSparse and (S.rows, S.cols) == (4, 4)
    assert same(S.toBreeze(), EXPECTED_TO_DENSE)
    assert same(suite_matrix().toDense(), EXPECTED_TO_DENSE)
    assert same(D.multiply(S).toBreeze(), EXPECTED_DENSE_SPARSE)
    assert same(S.multiply(S).toBreeze(), EXPECTED_SPARSE_SPARSE)
    assert same(suite_matrix().multiply(suite_matrix()), EXPECTED_SPARSE_SPARSE)
    assert same(S.multiply(D).toBreeze(), EXPECTED_SPARSE_DENSE)
    assert same(S.multiply(DENSE).toBreeze(), EXPECTED_SPARSE_DENSE)           # multiply(other: BDM) :107-119


SHAPES = [(1, 1, 1), (7, 5, 3), (33, 40, 35), (257, 513, 129), (1000, 999, 301)]
DENSITIES = [0.0, 1e-3, 1e-2, 0.1, 0.5]


@pytest.mark.parametrize("density", DENSITIES)
@pytest.mark.parametrize("m,k,n", SHAPES)
def test_kernels_bit_identical_to_the_reference_loops(m, k, n, density):
    rng = np.random.default_rng(hash((m, k, n, density)) % 2**32)
    A = so.random_csc(rng, m, k, density, empty_cols=0.1)
    B = so.random_csc(rng, k, n, density, empty_cols=0.1)
    Dl, Dr = rng.standard_normal((m, k)), rng.standard_normal((k, n))
    sA, sB = sp(A), sp(B)
    assert same(sA.toBreeze(), so.to_dense(A))
    assert same(mb.SubMatrix(Dl).multiply(sB).toBreeze(), so.mult_dense_sparse(Dl, B))
    assert same(sA.multiply(mb.SubMatrix(Dr)).toBreeze(), so.mult_sparse_dense(A, Dr))
    assert same(sA.multiply(sB).toBreeze(), so.spgemm(A, B))


def test_large_ragged_shape():
    rng = np.random.default_rng(11)
    m, k, n = 4096, 4093, 257
    A, B = so.random_csc(rng, m, k, 1e-3), so.random_csc(rng, k, n, 1e-2, empty_cols=0.3)
    Dl, Dr = rng.standard_normal((m, k)), rng.standard_normal((k, n))
    sA, sB = sp(A), sp(B)
    assert same(mb.SubMatrix(Dl).multiply(sB).toBreeze(), so.mult_dense_sparse(Dl, B))
    assert same(sA.multiply(mb.SubMatrix(Dr)).toBreeze(), so.mult_sparse_dense(A, Dr))
    assert same(sA.multiply(sB).toBreeze(), so.spgemm(A, B))
    assert same(sA.toBreeze(), so.to_dense(A))


def test_empty_blocks():
    rng = np.random.default_rng(2)
    for m, k, n in [(0, 5, 4), (5, 0, 4), (5, 4, 0), (0, 0, 0)]:
        A, B = so.random_csc(rng, m, k, 0.5), so.random_csc(rng, k, n, 0.5)
        Dl, Dr = rng.standard_normal((m, k)), rng.standard_normal((k, n))
        assert same(sp(A).multiply(sp(B)).toBreeze(), np.zeros((m, n)))
        assert same(mb.SubMatrix(Dl).multiply(sp(B)).toBreeze(), so.mult_dense_sparse(Dl, B))
        assert same(sp(A).multiply(mb.SubMatrix(Dr)).toBreeze(), so.mult_sparse_dense(A, Dr))


def test_special_values_and_the_copy_case():
    """Columns holding exactly one 1.0 copy the A column (keeping -0.0); explicit zeros, -0.0, inf and NaN are stored."""
    rng = np.random.default_rng(4)
    m, k, n = 37, 12, 9
    vals = rng.standard_normal((k, n))
    vals[:, 0] = 0.0
    vals[3, 0] = 1.0                                               # column 0: a single stored 1.0 -> copy of A(:, 3)
    vals[5, 1] = -0.0
    vals[6, 2] = np.inf
    mask = rng.random((k, n)) < 0.4
    mask[:, 0] = False
    mask[3, 0] = True
    mask[5, 1] = mask[6, 2] = mask[7, 3] = True
    vals[7, 3] = 0.0                                               # explicit zero
    B = so.csc_from_dense_pattern(vals, mask)
    Dl = rng.standard_normal((m, k))
    Dl[:, 3] = -0.0
    Dl[0, 6] = np.nan
    got = mb.SubMatrix(Dl).multiply(sp(B)).toBreeze()
    ref = so.mult_dense_sparse(Dl, B)
    assert same(got, ref) and np.all(np.signbit(got[:, 0]))
    A = so.csc_from_dense_pattern(Dl, rng.random((m, k)) < 0.5)
    Dr = vals.copy()
    assert same(sp(A).multiply(mb.SubMatrix(Dr)).toBreeze(), so.mult_sparse_dense(A, Dr))
    assert same(sp(A).multiply(sp(B)).toBreeze(), so.spgemm(A, B))


def test_dense_operands_as_views():
    rng = np.random.default_rng(6)
    m, k, n = 65, 70, 33
    A, B = so.random_csc(rng, m, k, 0.1), so.random_csc(rng, k, n, 0.1)
    big = rng.standard_normal((200, 150))
    left = mb.SubMatrix(big).slice(10, 10 + m, 20, 20 + k)              # a slice: offset + ld
    assert same(left.multiply(sp(B)).toBreeze(), so.mult_dense_sparse(big[10:10 + m, 20:20 + k], B))
    right = mb.SubMatrix(big).slice(3, 3 + k, 5, 5 + n)
    assert same(sp(A).multiply(right).toBreeze(), so.mult_sparse_dense(A, big[3:3 + k, 5:5 + n]))
    Xt = rng.standard_normal((n, k))
    tview = mb.SubMatrix(Xt).t                                           # a transposed view
    assert same(sp(A).multiply(tview).toBreeze(), so.mult_sparse_dense(A, Xt.T))
    Yt = rng.standard_normal((k, m))
    assert same(mb.SubMatrix(Yt).t.multiply(sp(B)).toBreeze(), so.mult_dense_sparse(Yt.T, B))
    # a transposed output view
    out = mb.SubMatrix.zeros(n, m).t
    sp(A).multiply(mb.SubMatrix(Xt.T.copy()), out=out)
    assert same(out.toBreeze(), so.mult_sparse_dense(A, Xt.T))


def test_accumulate_is_c_plus_p():
    rng = np.random.default_rng(8)
    m, k, n = 90, 80, 70
    A, B = so.random_csc(rng, m, k, 0.05, empty_cols=0.2), so.random_csc(rng, k, n, 0.05, empty_cols=0.2)
    Dl, Dr = rng.standard_normal((m, k)), rng.standard_normal((k, n))
    C0 = rng.standard_normal((m, n))
    C0[0, :] = -0.0
    for left, right, ref in [(mb.SubMatrix(Dl), sp(B), so.mult_dense_sparse(Dl, B)),
                             (sp(A), mb.SubMatrix(Dr), so.mult_sparse_dense(A, Dr)),
                             (sp(A), sp(B), so.spgemm(A, B))]:
        out = mb.SubMatrix(C0)
        left.multiply(right, out=out, accumulate=True)
        assert same(out.toBreeze(), C0 + ref)


def test_scalar_ops_change_only_the_stored_values():
    rng = np.random.default_rng(9)
    A = so.random_csc(rng, 50, 40, 0.2)
    s = sp(A)
    vals = mb.SubMatrix(A[4].reshape(-1, 1))
    for op, arg in [("add", 1.5), ("subtract", 0.25), ("divide", 3.0), ("multiply", -2.0)]:
        r = getattr(s, op)(arg)
        assert r.isSparse
        cp, ri, va = r.sparseBlock.to_host()
        assert np.array_equal(cp, A[2]) and np.array_equal(ri, A[3])
        assert same(va, getattr(vals, op)(arg).toBreeze().reshape(-1))
    assert same(s.add(1.0).toBreeze(), so.to_dense((A[0], A[1], A[2], A[3], A[4] + 1.0)))   # not A + 1


@pytest.mark.parametrize("seed", [1, 20260415, -7])
def test_generator_bit_identical_to_the_oracle(seed):
    n_rows, n_cols, by_row, by_col, d = 97, 61, 3, 2, 0.1
    m = MTUtils.randomBlockMatrix(None, n_rows, n_cols, by_row, by_col, (True, d), seed=seed)
    seeds = MTUtils._partition_seeds(seed, by_row * by_col)
    assert len(m.blocks) == by_row * by_col
    for b, blk in m.blocks:
        assert blk.isSparse
        rows, cols = blk.rows, blk.cols
        ref = so.sparse_block(seeds[b.row * by_col + b.column], rows, cols, so.column_count(cols, d))
        got = blk.sparseBlock.to_host()
        for x, y in zip(got, ref[2:]):
            assert np.array_equal(x, y)


def test_generator_large_block_properties():
    m = MTUtils.randomBlockMatrix(None, 4096, 4096, 1, 1, (True, 0.01), seed=3)
    cp, ri, va = m.blocks[0][1].sparseBlock.to_host()
    s = int(4096 * 0.01)
    assert np.array_equal(cp, np.arange(4097) * s)
    r = ri.reshape(4096, s)
    assert np.all(np.diff(r, axis=1) > 0) and r.min() >= 0 and r.max() < 4096
    assert np.all((va >= 0) & (va < 1))
    dense = MTUtils.randomBlockMatrix(None, 4096, 4096, 1, 1, seed=3)
    assert same(va, dense.blocks[0][1].toBreeze().reshape(-1, order="F")[: s * 4096])


def _grid(blocks_np, sparse_mask):
    out = []
    for (i, j), X in blocks_np.items():
        out.append((mb.BlockID(i, j), sp(X) if sparse_mask else mb.SubMatrix(X)))
    return out


def _split(rng, M, N, g, density, sparse):
    bm, bn = -(-M // g), -(-N // g)
    tiles = {}
    for i in range(g):
        for j in range(g):
            r, c = min(bm, M - i * bm), min(bn, N - j * bn)
            tiles[(i, j)] = so.random_csc(rng, r, c, density) if sparse else rng.standard_normal((r, c))
    return tiles


@pytest.mark.parametrize("g", [2, 3])
@pytest.mark.parametrize("kind", ["ss", "ds", "sd"])
def test_block_matrix_multiply_with_sparse_blocks(g, kind):
    rng = np.random.default_rng(g * 10 + len(kind))
    M, K, N = 301, 257, 199
    a_sp, b_sp = kind[0] == "s", kind[1] == "s"
    ta, tb = _split(rng, M, K, g, 0.05, a_sp), _split(rng, K, N, g, 0.05, b_sp)
    A = mb.BlockMatrix(_grid(ta, a_sp), M, K, g, g)
    B = mb.BlockMatrix(_grid(tb, b_sp), K, N, g, g)
    got = A.multiply(B)
    prod = {"ss": so.spgemm, "ds": so.mult_dense_sparse, "sd": so.mult_sparse_dense}[kind]
    for b, blk in got.blocks:
        ref = None
        for kk in range(g):
            p = prod(ta[(b.row, kk)], tb[(kk, b.column)])
            ref = p if ref is None else ref + p
        assert same(blk.toBreeze(), ref)                                     # C = P0 + P1 (+ P2), kk ascending
    dense = A.toDenseBlocks().multiply(B.toDenseBlocks()).toBreeze()
    assert np.abs(got.toBreeze() - dense).max() <= 1e-10 * max(1.0, np.abs(dense).max())


def test_multiply_local_matrix_and_multiply_by():
    rng = np.random.default_rng(12)
    M, K = 96, 96
    ta = _split(rng, M, K, 2, 0.1, True)
    A = mb.BlockMatrix(_grid(ta, True), M, K, 2, 2)
    Bl = rng.standard_normal((K, 50))
    got = A.multiply(Bl)                                                   # sparse x row-slice views of B (:280-303)
    for b, blk in got.blocks:
        ref = so.mult_sparse_dense(ta[(b.row, 0)], Bl[0:48]) + so.mult_sparse_dense(ta[(b.row, 1)], Bl[48:96])
        assert same(blk.toBreeze(), ref)
    Lb = rng.standard_normal((30, M))                                      # multiplyBy: local x sparse (:309-335)
    got = A.multiplyBy(Lb)
    for b, blk in got.blocks:
        ref = so.mult_dense_sparse(Lb[:, b.row * 48:(b.row + 1) * 48], ta[(b.row, b.column)])
        assert same(blk.toBreeze(), ref)


def test_to_dense_blocks_and_to_breeze():
    rng = np.random.default_rng(13)
    ta = _split(rng, 50, 40, 2, 0.2, True)
    A = mb.BlockMatrix(_grid(ta, True), 50, 40, 2, 2)
    full = np.zeros((50, 40))
    for (i, j), t in ta.items():
        full[i * 25:(i + 1) * 25, j * 20:(j + 1) * 20] = so.to_dense(t)
    assert same(A.toBreeze(), full)
    D = A.toDenseBlocks()
    assert not any(s.isSparse for _, s in D.blocks) and same(D.toBreeze(), full)
    assert same(D.toDenseBlocks().toBreeze(), full)                          # dense blocks are kept


def test_error_messages():
    S, D = mb.SubMatrix(spMatrix=suite_matrix()), mb.SubMatrix(DENSE)
    with pytest.raises(nat.MarlinArgumentError, match="Not supported add-operator between matrices of sparsity with true and false"):
        S.add(D)
    with pytest.raises(nat.MarlinArgumentError, match="Not supported subtract-operator between matrices of sparsity with false and true"):
        D.subtract(S)
    with pytest.raises(nat.MarlinArgumentError, match="call toDenseBlocks first"):
        S.denseBlock
    rng = np.random.default_rng(1)
    A = mb.BlockMatrix(_grid(_split(rng, 40, 40, 2, 0.2, True), True), 40, 40, 2, 2)
    for fn in (lambda: A.transpose(), lambda: A.add(A), lambda: A.sum(), lambda: A.toBlockMatrix(4, 4),
               lambda: A.toDenseVecMatrix()):
        with pytest.raises(nat.MarlinArgumentError, match="sparse blocks: call toDenseBlocks first") as e:
            fn()
        assert e.value.code == nat.MB_ERR_UNSUPPORTED
    with pytest.raises(nat.MarlinArgumentError, match="sparsity with true and vector"):
        mb.BlockMatrix(_grid(_split(rng, 40, 40, 1, 0.2, True), True), 40, 40, 1, 1).multiply(np.ones(40))
    with pytest.raises(nat.MarlinArgumentError, match="must be positive"):
        MTUtils.randomBlockMatrix(None, 10, 10, 1, 1, (True, 0.0), seed=1)
    with pytest.raises(nat.MarlinArgumentError, match="non-zeros per column asked"):
        MTUtils.randomBlockMatrix(None, 10, 200, 1, 1, (True, 0.1), seed=1)
    with pytest.raises(nat.MarlinArgumentError, match="distribution"):
        MTUtils.randomBlockMatrix(None, 10, 10, 1, 1, (True, 0.1), distribution=UniformGenerator(0, 2), seed=1)


def test_freivalds_16384_sparse_product():
    """A 16384^2 sparse x sparse product on a 2 x 2 grid at density 1e-3 (C is 2 GiB dense), checked by C x = A (B x)."""
    import scipy.sparse as sps
    A = MTUtils.randomBlockMatrix(None, 16384, 16384, 2, 2, (True, 1e-3), seed=5)
    B = MTUtils.randomBlockMatrix(None, 16384, 16384, 2, 2, (True, 1e-3), seed=6)
    Cm = A.multiply(B)

    def host(bm):
        rows = []
        for i in range(2):
            row = []
            for j in range(2):
                blk = dict(((b.row, b.column), s) for b, s in bm.blocks)[(i, j)]
                cp, ri, va = blk.sparseBlock.to_host()
                row.append(sps.csc_matrix((va, ri, cp), shape=(blk.rows, blk.cols)))
            rows.append(row)
        return sps.bmat(rows, format="csr")

    x = np.random.default_rng(0).standard_normal(16384)
    ref = host(A) @ (host(B) @ x)
    xt = torch.from_numpy(x).cuda()
    y = torch.zeros(16384, dtype=torch.float64, device="cuda")
    for b, blk in Cm.blocks:
        tile = blk.buf[: blk.rows * blk.cols].view(blk.cols, blk.rows).T
        y[b.row * 8192:(b.row + 1) * 8192] += tile @ xt[b.column * 8192:(b.column + 1) * 8192]
    got = y.cpu().numpy()
    assert np.abs(got - ref).max() <= 1e-9 * max(1.0, np.abs(ref).max())

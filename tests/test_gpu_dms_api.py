"""The DistributedMatrix API that completes the interface, on the GPU: the reference suite's "slice the matrix" and "repeat
by row and column" cases, cBind / repeat on both matrix types and every branch (including block grids that relabelling
would leave non-uniform), elementMultiply, zeros / ones, every `require` message, and the one-pass norm kernel
(mb_block_norm) against tests/dms_api_oracle.py: bit-exact where the arithmetic is a fixed fold, scaled entries, NaN and
Inf, strided views, large and wide shards, run-to-run bits, launch counts and the C ABI's errors; and two ranks against
one."""
import ctypes as C
import math
import os
import socket
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from tests import dms_api_oracle as do
from tests import marlin_cases as mc

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
A = mc.EXPECTED_DENSE


@pytest.fixture(scope="module")
def M():
    import marlin_b200 as mb
    mb.Runtime.get()
    return mb


def dvm(M, a=None, ids=None):
    if a is None:
        return M.DenseVecMatrix([(i, np.array(v)) for i, v in mc.DATA_ROWS])
    ids = range(a.shape[0]) if ids is None else ids
    return M.DenseVecMatrix([(int(i), a[int(i)]) for i in ids], a.shape[0], a.shape[1])


def blk(M, a, br, bc):
    return dvm(M, a).toBlockMatrix(br, bc)


def ints(m, n, seed, lo=-8, hi=8):
    return np.random.default_rng(seed).integers(lo, hi + 1, size=(m, n)).astype(np.float64)


def raises(M, call, msg):
    with pytest.raises(M.MarlinArgumentError) as e:
        call()
    assert str(e.value) == msg


# ---------------------------------------------------------------------------------------------- the suite cases
def test_slice_the_matrix(M):                           # DMS.scala:207-223
    mat = dvm(M)
    assert np.array_equal(mat.sliceByRow(1, 2).toBreeze(), np.array([[2.0, 3.0, 4.0, 5.0], [3.0, 2.0, 1.0, 0.0]]))
    assert np.array_equal(mat.sliceByColumn(1, 2).toBreeze(), np.array([[1.0, 2.0], [3.0, 4.0], [2.0, 1.0], [1.0, 1.0]]))
    assert np.array_equal(mat.getSubMatrix(1, 2, 1, 2).toBreeze(), np.array([[3.0, 4.0], [2.0, 1.0]]))


def test_repeat_by_row_and_column(M):                   # DMS.scala:354-374
    mat = dvm(M)
    assert np.array_equal(M.MTUtils.repeatByRow(mat, 2).toBreeze(), do.repeat_by_row(A, 2))
    assert np.array_equal(M.MTUtils.repeatByColumn(mat, 2).toBreeze(), do.repeat_by_column(A, 2))


# ---------------------------------------------------------------------------------------------- slicing
def test_slices_shift_ids_and_keep_ranks(M):
    a = ints(37, 11, 1)
    mat = dvm(M, a, ids=np.random.default_rng(2).permutation(37))
    s = mat.sliceByRow(5, 20)
    assert (s.numRows(), s.numCols()) == (16, 11) and sorted(s.ids.tolist()) == list(range(16))
    assert np.array_equal(s.toBreeze(), a[5:21])
    assert np.array_equal(mat.sliceByColumn(3, 3).toBreeze(), a[:, 3:4])
    assert np.array_equal(mat.getSubMatrix(36, 36, 0, 10).toBreeze(), a[36:37])
    assert np.array_equal(mat.getSubMatrix(2, 30, 4, 9).toBreeze(), do.get_sub_matrix(a, 2, 30, 4, 9))


def test_slice_requires(M):
    mat = dvm(M)
    row = "start row or end row mismatch the matrix num of rows"
    col = "start column or end column mismatch the matrix num of columns"
    for call in (lambda: mat.sliceByRow(-1, 2), lambda: mat.sliceByRow(1, 4), lambda: mat.sliceByRow(3, 2)):
        raises(M, call, row)
    for call in (lambda: mat.sliceByColumn(-1, 2), lambda: mat.sliceByColumn(0, 4), lambda: mat.sliceByColumn(2, 1)):
        raises(M, call, col)
    for call in (lambda: mat.getSubMatrix(-1, 1, 0, 1), lambda: mat.getSubMatrix(0, 4, 0, 1), lambda: mat.getSubMatrix(2, 1, 0, 1)):
        raises(M, call, "start row or end row dismatch the matrix num of rows")
    for call in (lambda: mat.getSubMatrix(0, 1, -1, 1), lambda: mat.getSubMatrix(0, 1, 0, 4), lambda: mat.getSubMatrix(0, 1, 3, 2)):
        raises(M, call, "start column or end column dismatch the matrix num of columns")


# ---------------------------------------------------------------------------------------------- cBind
def test_dense_cbind(M):
    a, b = ints(9, 5, 3), ints(9, 4, 4)
    got = dvm(M, a).cBind(dvm(M, b, ids=np.arange(9)[::-1]))
    assert isinstance(got, M.DenseVecMatrix) and (got.numRows(), got.numCols()) == (9, 9)
    assert np.array_equal(got.toBreeze(), np.hstack([a, b]))
    got = dvm(M, a).cBind(blk(M, b, 2, 2))                                 # a BlockMatrix goes through its rows
    assert np.array_equal(got.toBreeze(), np.hstack([a, b]))


def test_dense_cbind_is_an_inner_join(M):
    a, b = ints(6, 3, 5), ints(6, 2, 6)
    got = dvm(M, a).cBind(dvm(M, b, ids=[0, 2, 3, 5]))
    assert sorted(got.ids.tolist()) == [0, 2, 3, 5] and (got.numRows(), got.numCols()) == (6, 5)
    rows = do.cbind_rows({i: a[i] for i in range(6)}, {i: b[i] for i in (0, 2, 3, 5)})
    for pos, i in enumerate(got.ids):
        assert np.array_equal(got.data.toBreeze()[pos], rows[int(i)])


def test_cbind_errors(M):
    from marlin_b200.matrix.distributed_matrix import DistributedMatrix

    class Other(DistributedMatrix):
        def numRows(self):
            return 4

    mat, five = dvm(M), dvm(M, ints(5, 4, 7))
    raises(M, lambda: mat.cBind(five), "Dimension mismatch:  4 vs 5")
    raises(M, lambda: mat.cBind(Other()), f"Do not support this type {Other} for cBind operation")
    bm = blk(M, A, 2, 2)
    raises(M, lambda: bm.cBind(blk(M, ints(5, 4, 7), 2, 2)), "Row dimension mismatches: 4 vs 5")
    raises(M, lambda: bm.cBind(Other()), "have not implemented yet")


def test_block_cbind_relabels_in_place(M):
    a, b = ints(8, 6, 8), ints(8, 6, 9)
    x, y = blk(M, a, 2, 2), blk(M, b, 2, 2)
    got = x.cBind(y)
    assert isinstance(got, M.BlockMatrix)
    assert (got.numRows(), got.numCols(), got.numBlksByRow(), got.numBlksByCol()) == (8, 12, 2, 4)
    held = {(k.row, k.column): s for k, s in got.blocks}
    for k, s in y.blocks:
        assert held[(k.row, k.column + 2)] is s                             # no block copied
    assert np.array_equal(got.toBreeze(), np.hstack([a, b]))
    assert np.array_equal(got.toDenseVecMatrix().toBreeze(), np.hstack([a, b]))


@pytest.mark.parametrize("shapes", [((4, 5), (2, 2), (4, 4), (2, 2)),       # widths 3,2 + 2,2: the grid of 9 is 3,3,3,0
                                    ((4, 4), (2, 2), (4, 3), (1, 3)),       # different block-row counts
                                    ((6, 4), (3, 2), (6, 3), (3, 1))])      # widths 2,2 + 3: the grid of 7 in 3 is 3,3,1
def test_block_cbind_takes_the_rows_route(M, shapes):
    (ma, na), (bra, bca), (mb_, nb), (brb, bcb) = shapes
    a, b = ints(ma, na, 10), ints(mb_, nb, 11)
    got = blk(M, a, bra, bca).cBind(blk(M, b, brb, bcb))
    assert isinstance(got, M.DenseVecMatrix)
    assert np.array_equal(got.toBreeze(), np.hstack([a, b]))
    got = blk(M, a, bra, bca).cBind(dvm(M, b))
    assert isinstance(got, M.DenseVecMatrix) and np.array_equal(got.toBreeze(), np.hstack([a, b]))


# ---------------------------------------------------------------------------------------------- repeat
@pytest.mark.parametrize("times", [1, 2, 3])
def test_dense_repeat(M, times):
    a = ints(7, 5, 12)
    mat = dvm(M, a)
    r, c = M.MTUtils.repeatByRow(mat, times), M.MTUtils.repeatByColumn(mat, times)
    if times == 1:
        assert r is mat and c is mat
    assert (r.numRows(), r.numCols(), c.numRows(), c.numCols()) == (7, 5 * times, 7 * times, 5)
    assert np.array_equal(r.toBreeze(), do.repeat_by_row(a, times))
    assert np.array_equal(c.toBreeze(), do.repeat_by_column(a, times))


@pytest.mark.parametrize("times", [1, 2, 3])
@pytest.mark.parametrize("shape", [(8, 6, 2, 2), (4, 5, 2, 2), (5, 4, 2, 2), (9, 9, 3, 3)])
def test_block_repeat(M, shape, times):
    m, n, br, bc = shape
    a = ints(m, n, 13)
    bm = blk(M, a, br, bc)
    r, c = M.MTUtils.repeatByRow(bm, times), M.MTUtils.repeatByColumn(bm, times)
    if times == 1:
        assert r is bm and c is bm
    assert isinstance(r, M.BlockMatrix) and isinstance(c, M.BlockMatrix)
    assert (r.numRows(), r.numCols(), c.numRows(), c.numCols()) == (m, n * times, m * times, n)
    assert np.array_equal(r.toBreeze(), do.repeat_by_row(a, times))
    assert np.array_equal(c.toBreeze(), do.repeat_by_column(a, times))
    assert np.array_equal(r.toDenseVecMatrix().toBreeze(), do.repeat_by_row(a, times))
    relabelled = do.relabel_keeps_grid(do.extents(n, bc) * times)
    if times > 1 and relabelled:
        held = {id(s) for _, s in bm.blocks}
        assert all(id(s) in held for _, s in r.blocks) and r.numBlksByCol() == bc * times


def test_repeat_requires(M):
    for t in (0, -1):
        raises(M, lambda: M.MTUtils.repeatByRow(dvm(M), t), f"repeat times: {t} illegal")
        raises(M, lambda: M.MTUtils.repeatByColumn(blk(M, A, 2, 2), t), f"repeat times: {t} illegal")


# ---------------------------------------------------------------------------------------------- elementMultiply
def test_element_multiply(M):
    a, b = ints(9, 7, 14), ints(9, 7, 15)
    x, y = blk(M, a, 3, 2), blk(M, b, 3, 2)
    got = x.elementMultiply(y, None)
    assert np.array_equal(got.toBreeze(), a * b)
    assert np.array_equal(x.toBreeze(), a) and np.array_equal(y.toBreeze(), b)         # this is unchanged
    assert np.array_equal(x.elementMultiply(y).toBreeze(), a * b)
    part = M.BlockMatrix([(k, s) for k, s in y.blocks if (k.row, k.column) != (1, 1)], 9, 7, 3, 2)
    got = x.elementMultiply(part, object())
    want = do.element_multiply({(k.row, k.column): s.toBreeze() for k, s in x.blocks},
                               {(k.row, k.column): s.toBreeze() for k, s in part.blocks})
    assert {(k.row, k.column) for k, _ in got.blocks} == set(want)
    for k, s in got.blocks:
        assert np.array_equal(s.toBreeze(), want[(k.row, k.column)])


def test_element_multiply_sparse_raises(M):
    sp = M.MTUtils.randomBlockMatrix(None, 8, 8, 2, 2, sparseInfo=(True, 0.5), seed=3)
    with pytest.raises(M.MarlinArgumentError, match="not supported on sparse blocks"):
        sp.elementMultiply(blk(M, ints(8, 8, 1), 2, 2))


# ---------------------------------------------------------------------------------------------- zeros / ones
def test_zeros_and_ones(M):
    z = M.MTUtils.zerosDenVecMatrix(None, 11, 6)
    o = M.MTUtils.onesDenVecMatrix(None, 11, 6)
    r = M.MTUtils.randomDenVecMatrix(None, 11, 6, seed=1)
    assert np.array_equal(z.toBreeze(), do.constant(11, 6, 0.0)) and np.array_equal(o.toBreeze(), do.constant(11, 6, 1.0))
    assert z.ids.tolist() == r.ids.tolist() == o.ids.tolist()
    assert (o.numRows(), o.numCols()) == (11, 6)


# ---------------------------------------------------------------------------------------------- norms
def _bits(x):
    return np.float64(x).view(np.int64)


def test_norms_of_the_suite_matrix(M):
    mat = dvm(M)
    assert mat.norm("1") == 9.0 and mat.norm("inf") == 14.0 and mat.norm("fro") == math.sqrt(float((A * A).sum()))
    neg = dvm(M, -A)
    assert neg.norm("inf") == 14.0 and neg.norm("1") == 9.0
    for mode in ("2", "Inf", "for", ""):
        raises(M, lambda: mat.norm(mode), f"Do not support mode {mode}.")


@pytest.mark.parametrize("shape", [(1, 1), (31, 33), (1000, 300), (4097, 65), (5000, 7)])
def test_inf_is_the_sequential_fold_bit_for_bit(M, shape):
    a = np.random.default_rng(sum(shape)).standard_normal(shape) * 10.0 ** np.random.default_rng(1).integers(-3, 4, size=shape)
    want = np.cumsum(np.abs(a), axis=1)[:, -1].max()
    assert _bits(dvm(M, a).norm("inf")) == _bits(want)


@pytest.mark.parametrize("shape", [(1, 1), (31, 33), (4097, 65), (9000, 130)])
def test_one_and_fro_exact_on_integers(M, shape):
    a = ints(*shape, seed=shape[0])
    mat = dvm(M, a)
    assert mat.norm("1") == np.abs(a).sum(axis=0).max()
    assert mat.norm("fro") == math.sqrt(float((a * a).sum()))


@pytest.mark.parametrize("shape", [(3000, 200), (10000, 33)])
def test_random_data_within_rounding(M, shape):
    a = np.random.default_rng(5).standard_normal(shape)
    mat = dvm(M, a)
    tol = shape[0] * 2.0 ** -53
    assert mat.norm("1") == pytest.approx(do.norm(a, "1"), rel=tol, abs=0)
    assert mat.norm("fro") == pytest.approx(do.norm(a, "fro"), rel=tol, abs=0)


@pytest.mark.parametrize("scale", [1e300, 1e-300, 5e-324, 2.0 ** -1060, 1e154, 1e-154])
def test_fro_without_spurious_overflow_or_underflow(M, scale):
    a = ints(300, 40, 16, lo=1, hi=9) * scale
    got = dvm(M, a).norm("fro")
    assert math.isfinite(got) and got > 0.0
    assert got == pytest.approx(do.norm(a, "fro"), rel=1e-13)
    mixed = ints(50, 20, 17)
    mixed[3, 4], mixed[7, 1] = 1e300, 5e-324
    assert dvm(M, mixed).norm("fro") == pytest.approx(do.norm(mixed, "fro"), rel=1e-14)
    tiny = np.full((10, 10), 5e-324)
    tiny[0, 0] = 1.0                                       # small and medium together
    assert dvm(M, tiny).norm("fro") == 1.0


def test_nan_and_inf(M):
    for poison, expect_nan in ((math.nan, True), (math.inf, False), (-math.inf, False)):
        a = ints(100, 50, 18)
        a[40, 7] = poison
        mat = dvm(M, a)
        for mode in ("1", "inf", "fro"):
            got = mat.norm(mode)
            assert (math.isnan(got) if expect_nan else got == math.inf), (poison, mode, got)
    a = ints(100, 50, 19)
    a[3, 3], a[90, 40] = math.inf, math.nan
    for mode in ("1", "inf", "fro"):
        assert math.isnan(dvm(M, a).norm(mode))


def test_empty_matrix(M):
    empty = M.DenseVecMatrix(ids=np.zeros(0, np.int64), data=None, nRows=3, nCols=4)
    for mode in ("1", "inf", "fro"):
        with pytest.raises(M.MarlinError) as e:
            empty.norm(mode)
        assert e.value.code == M._native.MB_ERR_EMPTY and "empty collection" in str(e.value)


def _strided(M, a, ld_extra, row_major):
    """`a` as a view with a leading dimension larger than its rows (column-major) or columns (row-major)."""
    import torch
    m, n = a.shape
    if row_major:
        host = np.full((m, n + ld_extra), 7.0)
        host[:, :n] = a
        buf = torch.from_numpy(host.reshape(-1).copy()).cuda()
        return M.SubMatrix(buf=buf, rows=m, cols=n, ld=n + ld_extra, is_transpose=True)
    host = np.full((n, m + ld_extra), 7.0)
    host[:, :m] = a.T
    buf = torch.from_numpy(host.reshape(-1).copy()).cuda()
    return M.SubMatrix(buf=buf, rows=m, cols=n, ld=m + ld_extra, is_transpose=False)


@pytest.mark.parametrize("row_major", [True, False])
def test_strided_views(M, row_major):
    a = np.random.default_rng(20).standard_normal((333, 45))
    view = _strided(M, a, 9, row_major)
    mat = M.DenseVecMatrix(ids=np.arange(333), data=view, nRows=333, nCols=45)
    assert _bits(mat.norm("inf")) == _bits(np.cumsum(np.abs(a), axis=1)[:, -1].max())
    assert mat.norm("1") == pytest.approx(do.norm(a, "1"), rel=1e-13)
    assert mat.norm("fro") == pytest.approx(do.norm(a, "fro"), rel=1e-13)
    sub = _strided(M, a, 9, row_major).slice(10, 300, 3, 40)                    # an offset view
    smat = M.DenseVecMatrix(ids=np.arange(290), data=sub, nRows=290, nCols=37)
    assert _bits(smat.norm("inf")) == _bits(np.cumsum(np.abs(a[10:300, 3:40]), axis=1)[:, -1].max())


def test_large_shard(M):
    import torch
    rt = M.Runtime.get()
    m, n = 1 << 20, 1024
    buf = torch.randint(-3, 4, (m * n,), dtype=torch.int8, device=rt.device).to(torch.float64)
    mat = M.DenseVecMatrix(ids=np.arange(m), data=M.SubMatrix(buf=buf, rows=m, cols=n, ld=n, is_transpose=True), nRows=m, nCols=n)
    t = buf.view(m, n).abs()
    assert mat.norm("inf") == float(t.sum(dim=1).max())
    assert mat.norm("1") == float(t.sum(dim=0).max())
    assert mat.norm("fro") == math.sqrt(float((t * t).sum()))
    del t


def test_odd_wide_shard(M):
    a = np.random.default_rng(21).standard_normal((300, 100003))
    mat = dvm(M, a)
    assert _bits(mat.norm("inf")) == _bits(np.cumsum(np.abs(a), axis=1)[:, -1].max())
    assert mat.norm("1") == pytest.approx(do.norm(a, "1"), rel=300 * 2.0 ** -53)
    assert mat.norm("fro") == pytest.approx(do.norm(a, "fro"), rel=1e-12)


def test_run_to_run_bits(M):
    a = np.random.default_rng(22).standard_normal((20000, 333))
    mat = dvm(M, a)
    for mode in ("1", "inf", "fro"):
        first = mat.norm(mode)
        assert all(_bits(mat.norm(mode)) == _bits(first) for _ in range(3))


def test_launch_count_and_errors(M):
    import torch
    nat = M._native
    rt = M.Runtime.get()
    a = dvm(M, ints(5000, 70, 23))
    col = M.SubMatrix.empty(70, 1, nat.MB_F64)
    out = np.zeros(3)
    for kind, launches in ((nat.MB_NORM_ONE, 2), (nat.MB_NORM_INF, 1), (nat.MB_NORM_FRO, 2)):
        rt.sync_stream()
        before = rt.lib.mb_launch_count(rt.ctx)
        nat.check(rt.lib.mb_block_norm(rt.ctx, a.data.handle(), kind, col.handle(), out.ctypes.data_as(nat.c_dp)))
        assert rt.lib.mb_launch_count(rt.ctx) - before == launches
        if kind == nat.MB_NORM_ONE:
            assert out[0] == np.abs(a.data.toBreeze()).sum(axis=0).max()
            assert np.array_equal(col.toBreeze().reshape(-1), np.abs(a.data.toBreeze()).sum(axis=0))
    short = M.SubMatrix.empty(69, 1, nat.MB_F64)
    assert rt.lib.mb_block_norm(rt.ctx, a.data.handle(), nat.MB_NORM_ONE, short.handle(), None) == nat.MB_ERR_DIM_MISMATCH
    assert rt.lib.mb_block_norm(rt.ctx, a.data.handle(), 7, None, out.ctypes.data_as(nat.c_dp)) == nat.MB_ERR_INVALID_ARG
    assert rt.lib.mb_block_norm(rt.ctx, a.data.handle(), nat.MB_NORM_INF, None, None) == nat.MB_ERR_INVALID_ARG
    bf = a.data.copy(nat.MB_BF16)
    assert rt.lib.mb_block_norm(rt.ctx, bf.handle(), nat.MB_NORM_INF, None, out.ctypes.data_as(nat.c_dp)) == nat.MB_ERR_UNSUPPORTED
    none = M.SubMatrix(buf=torch.zeros(0, dtype=torch.float64, device=rt.device), rows=0, cols=70, ld=70, is_transpose=True)
    assert rt.lib.mb_block_norm(rt.ctx, none.handle(), nat.MB_NORM_INF, None, out.ctypes.data_as(nat.c_dp)) == nat.MB_ERR_EMPTY


# ---------------------------------------------------------------------------------------------- two ranks
def test_two_ranks_match_one(M, tmp_path):
    sys.path.insert(0, str(ROOT / "tests"))
    import dms_api_gpu_worker as w
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    env = dict(os.environ, DMS_API_WORKER_OUT=str(tmp_path / "r"))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), str(ROOT / "tests" / "dms_api_gpu_worker.py")]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900, env=env)
    assert out.returncode == 0, out.stdout[-4000:]
    for r in range(2):
        assert f"rank {r} dms api ok" in out.stdout
    two = dict(np.load(str(tmp_path / "r.0.npz")))
    one = w.run(M)
    assert set(two) == set(one)
    for k in one:
        if k.startswith("norm_inf"):
            assert _bits(two[k]) == _bits(one[k]), k                        # the same bits for any number of ranks
        else:
            assert np.array_equal(two[k], one[k]), k

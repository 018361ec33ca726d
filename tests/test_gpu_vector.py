"""GPU parity of the vector side of the path (SURVEY 8f-4): mb_block_gemv / mb_block_dot / mb_block_ger through the
C ABI, and DistributedVector / BlockMatrix.multiply(vector) / DenseVecMatrix.multiply(vector) through the host mirror,
against the F2J-order oracle (dgemv.f / ddot.f) and the reference suite's own vectors (DistributedMatrixSuite.scala:
121-143, 390-409).

Tolerances: ger is BIT-EXACT (one IEEE multiply per element); a gemv whose contraction fits one column chunk (<= 256
columns, plain orientation) is BIT-EXACT with F2J's dgemv (same order, separate multiply and add); everything else
satisfies max_i |y - y_ref|_i / (|A||x|)_i <= 1e-10 (the north_star's fp64 bound).
"""
import ctypes as C

import numpy as np
import pytest

from marlin_b200 import _native as nat
from tests import marlin_cases as mc
from tests.harness import gpu  # noqa: F401  (a fixture)
from tests.test_gpu_cabi import alloc, download, upload, upload_mat

pytestmark = pytest.mark.gpu
TOL = 1e-10


def _scaled(got, ref, A, x):
    denom = np.abs(A) @ np.abs(x)
    denom[denom == 0] = 1.0
    return (np.abs(got - ref) / denom).max()


# ---------------------------------------------------------------------------------------- C ABI
@pytest.mark.parametrize("shape", [(1, 1), (2, 3), (4, 4), (50, 50), (100, 100), (255, 257), (256, 256), (257, 255),
                                   (513, 8), (7, 1000), (1000, 777), (2049, 1030), (301, 4099)])
@pytest.mark.parametrize("trans", [0, 1])
def test_gemv_vs_f2j_oracle(gpu, oracle, shape, trans):
    lib, ctx = gpu
    m, n = shape
    rng = np.random.default_rng(m * 131 + n + trans)
    A = rng.random((m, n)) * 2 - 1
    x = rng.random(n) * 2 - 1
    ref = oracle.block_multiply_vector(np.ascontiguousarray(A) if trans else np.asfortranarray(A), x)
    ha = upload(gpu, np.asfortranarray(A.T).reshape(-1, order="F"), 0, m, n, max(1, n), 1) if trans else upload_mat(gpu, A)
    hx = upload_mat(gpu, x.reshape(-1, 1))
    hy = alloc(gpu, m, 1)
    nat.check(lib.mb_block_gemv(ctx, ha, hx, hy, 0))
    got = download(gpu, hy, m, 1).reshape(-1)
    assert _scaled(got, ref, A, x) <= TOL
    if not trans and n <= 256:
        assert np.array_equal(got, ref)                      # same order as dgemv.f, no FMA: bit-exact
    nat.check(lib.mb_block_gemv(ctx, ha, hx, hy, 1))         # accumulate = the reduceByKey add (BlockMatrix.scala:251)
    got2 = download(gpu, hy, m, 1).reshape(-1)
    assert np.array_equal(got2, got + got)
    for h in (ha, hx, hy):
        lib.mb_block_free(ctx, h)


def test_gemv_strided_views_and_row_vectors(gpu, oracle):
    """Odd majorStride / odd offset (no 128-bit path), x and y given as single-row blocks, and the mb_block_gemm
    dispatch of the degenerate shapes (n x 1, 1 x n, k = 1) onto the vector kernels."""
    lib, ctx = gpu
    rng = np.random.default_rng(11)
    m, n, ld, off = 61, 45, 67, 3
    store = rng.random(off + ld * n)
    A = store[off:off + ld * n].reshape(n, ld).T[:m, :]
    x = rng.random(n)
    ha = upload(gpu, store, off, m, n, ld, 0)
    hx = upload(gpu, x, 0, 1, n, 1, 0)                       # a 1 x n row block
    hy = alloc(gpu, 1, m)
    nat.check(lib.mb_block_gemv(ctx, ha, hx, hy, 0))
    ref = oracle.block_multiply_vector(np.asfortranarray(A), x)
    assert np.array_equal(download(gpu, hy, 1, m).reshape(-1), ref)
    # mb_block_gemm with B = n x 1
    hx2 = upload_mat(gpu, x.reshape(-1, 1))
    hc = alloc(gpu, m, 1)
    nat.check(lib.mb_block_gemm(ctx, ha, hx2, hc, 0))
    assert np.array_equal(download(gpu, hc, m, 1).reshape(-1), ref)
    # row x matrix: (1 x m) . (m x n)
    w = rng.random(m)
    hw = upload(gpu, w, 0, 1, m, 1, 0)
    hr = alloc(gpu, 1, n)
    nat.check(lib.mb_block_gemm(ctx, hw, ha, hr, 0))
    got = download(gpu, hr, 1, n).reshape(-1)
    assert (np.abs(got - w @ A) / (np.abs(w) @ np.abs(A))).max() <= TOL
    # k = 1: column x row
    hcol = upload_mat(gpu, w.reshape(-1, 1))
    ho = alloc(gpu, m, n)
    nat.check(lib.mb_block_gemm(ctx, hcol, hx, ho, 0))
    assert np.array_equal(download(gpu, ho, m, n), np.outer(w, x))


@pytest.mark.parametrize("n", [1, 2, 5, 257, 2048, 2049, 100003, 1 << 21])
def test_dot_vs_oracle(gpu, oracle, n):
    lib, ctx = gpu
    rng = np.random.default_rng(n)
    x, y = rng.random(n) * 2 - 1, rng.random(n) * 2 - 1
    hx, hy = upload_mat(gpu, x.reshape(-1, 1)), upload_mat(gpu, y.reshape(-1, 1))
    out = C.c_double()
    nat.check(lib.mb_block_dot(ctx, hx, hy, C.byref(out)))
    ref = oracle.vector_dot(x, y)
    assert abs(out.value - ref) <= TOL * float(np.abs(x) @ np.abs(y))
    out2 = C.c_double()
    nat.check(lib.mb_block_dot(ctx, hx, hy, C.byref(out2)))
    assert out2.value == out.value                           # fixed grid and order: run-to-run reproducible
    for h in (hx, hy):
        lib.mb_block_free(ctx, h)


@pytest.mark.parametrize("shape", [(1, 1), (2, 2), (3, 7), (255, 9), (256, 8), (513, 130), (1000, 1001)])
def test_ger_bit_exact(gpu, oracle, shape):
    lib, ctx = gpu
    m, n = shape
    rng = np.random.default_rng(m + 7 * n)
    x, y = rng.random(m) * 2 - 1, rng.random(n) * 2 - 1
    hx, hy = upload_mat(gpu, x.reshape(-1, 1)), upload_mat(gpu, y.reshape(-1, 1))
    ho = alloc(gpu, m, n)
    nat.check(lib.mb_block_ger(ctx, hx, hy, ho))
    assert np.array_equal(download(gpu, ho, m, n), oracle.vector_outer(x, y))
    # transposed (row-major) result block
    hot = alloc(gpu, n, m)
    vt = nat.c_blk()
    nat.check(lib.mb_block_view_t(ctx, hot, C.byref(vt)))
    nat.check(lib.mb_block_ger(ctx, hx, hy, vt))
    assert np.array_equal(download(gpu, hot, n, m).T, np.outer(x, y))


def test_vector_error_codes(gpu):
    lib, ctx = gpu
    a = alloc(gpu, 4, 3)
    x3, x4, y4 = alloc(gpu, 3, 1), alloc(gpu, 4, 1), alloc(gpu, 4, 1)
    out = C.c_double()
    assert lib.mb_block_gemv(ctx, a, x4, y4, 0) == nat.MB_ERR_DIM_MISMATCH
    assert b"Dimension mismatch" in lib.mb_last_error()
    assert lib.mb_block_gemv(ctx, a, x3, x3, 0) == nat.MB_ERR_DIM_MISMATCH
    assert lib.mb_block_gemv(ctx, a, a, y4, 0) == nat.MB_ERR_UNSUPPORTED          # x is not a vector
    assert lib.mb_block_dot(ctx, x3, x4, C.byref(out)) == nat.MB_ERR_DIM_MISMATCH
    assert lib.mb_block_ger(ctx, x4, x3, x4) == nat.MB_ERR_DIM_MISMATCH
    assert lib.mb_block_gemv(ctx, None, x3, y4, 0) == nat.MB_ERR_INVALID_ARG


def test_full_size_gemv_properties(gpu):
    """16384 x 16384 (2 GiB) through size-independent properties: A . ones = row sums (checked against the sum kernel:
    a checksum of checksums), A^T-view . e_j = row j, linearity in x."""
    import torch
    lib, ctx = gpu
    n = 16384
    p = lambda t: C.c_void_p(t.data_ptr())
    g = torch.Generator(device="cuda"); g.manual_seed(7)
    A = torch.rand(n * n, dtype=torch.float64, device="cuda", generator=g)
    x = torch.rand(n, dtype=torch.float64, device="cuda", generator=g)
    ones = torch.ones(n, dtype=torch.float64, device="cuda")
    y = torch.empty(n, dtype=torch.float64, device="cuda")
    y2 = torch.empty(n, dtype=torch.float64, device="cuda")

    def wrap(t, rows, cols, ld, trans=0):
        h = nat.c_blk()
        nat.check(lib.mb_block_wrap(ctx, p(t), 0, rows, cols, ld, trans, nat.MB_F64, C.byref(h)))
        return h
    ha, hat = wrap(A, n, n, n), wrap(A, n, n, n, 1)
    hx, h1, hy, hy2 = wrap(x, n, 1, n), wrap(ones, n, 1, n), wrap(y, n, 1, n), wrap(y2, n, 1, n)
    nat.check(lib.mb_set_stream(ctx, None))
    nat.check(lib.mb_block_gemv(ctx, ha, h1, hy, 0))
    total = C.c_double()
    nat.check(lib.mb_block_sum(ctx, ha, C.byref(total)))
    nat.check(lib.mb_synchronize(ctx))
    assert abs(float(y.sum()) - total.value) <= 1e-12 * total.value
    Am = A.view(n, n)                                        # Am[c, r] = A(r, c)
    assert torch.allclose(y, Am.sum(dim=0), rtol=1e-12, atol=0)
    # transposed view: y = A^T x
    nat.check(lib.mb_block_gemv(ctx, hat, hx, hy, 0))
    nat.check(lib.mb_synchronize(ctx))
    assert torch.allclose(y, Am @ x, rtol=1e-11, atol=0)
    # linearity: A(x + 1) = A x + A 1
    nat.check(lib.mb_block_gemv(ctx, ha, hx, hy, 0))
    nat.check(lib.mb_block_gemv(ctx, ha, h1, hy, 1))
    xp1 = x + 1.0
    nat.check(lib.mb_block_gemv(ctx, ha, wrap(xp1, n, 1, n), hy2, 0))
    nat.check(lib.mb_synchronize(ctx))
    assert torch.allclose(y, y2, rtol=1e-12, atol=0)
    nat.check(lib.mb_reset_stream(ctx))


# ---------------------------------------------------------------------------------------- host mirror
@pytest.fixture(scope="module")
def M():
    import marlin_b200 as mb
    mb.Runtime.get()
    return mb


def test_disvec_to_disvec(M):                             # DistributedMatrixSuite.scala:121-143
    v1 = M.DistributedVector([(i, np.array(v)) for i, v in mc.DISVEC_PIECES])
    v2 = v1.toDisVector(mc.DISVEC_SPLIT_STATUS, 4)
    assert v2.splitNum == 4 and all(p.rows == 3 for _, p in v2.vectors)
    assert np.array_equal(v1.toBreeze(), v2.toBreeze())
    assert np.array_equal(v2.toBreeze(), np.arange(12.0))


def test_blas1_distributed_vector(M):                     # DistributedMatrixSuite.scala:390-409
    pieces = [(i, np.array(v)) for i, v in mc.BLAS1_PIECES]
    v1, v2 = M.DistributedVector(pieces), M.DistributedVector(pieces)
    mat = v1.multiply(v2.transpose())
    assert isinstance(mat, M.BlockMatrix) and np.array_equal(mat.toBreeze(), mc.BLAS1_OUTER)
    assert v1.transpose().multiply(v2) == mc.BLAS1_INNER
    assert v1.transpose().multiply(v2, "local") == mc.BLAS1_INNER
    with pytest.raises(ValueError):
        v1.multiply(v2)
    with pytest.raises(ValueError):
        v1.transpose().multiply(v2, "elsewhere")
    d = v1.substract(v2)
    assert np.array_equal(d.toBreeze(), np.zeros(4))


def test_matrix_vector_golden(M):
    """The suite's 4 x 4 matrix times [1,2,3,4] through every overload (exact, small integers)."""
    x = np.array(mc.MATVEC_X)
    ma = M.BlockMatrix([(M.BlockID(*k), M.SubMatrix(np.array(v))) for k, v in mc.BLKS])
    mat = M.DenseVecMatrix([(i, np.array(v)) for i, v in mc.DATA_ROWS])
    dv = M.DistributedVector.fromVector(None, x, 2)
    assert np.array_equal(ma.multiply(dv).toBreeze(), mc.MATVEC_Y)
    assert np.array_equal(mat.multiply(dv, (2, 2)).toBreeze(), mc.MATVEC_Y)
    assert np.array_equal(mat.multiply(x, 2).toBreeze(), mc.MATVEC_Y)
    assert np.array_equal(mat.multiply(x), mc.MATVEC_Y)
    with pytest.raises(ValueError):
        ma.multiply(x)                                    # "should not split the matrix by column"
    with pytest.raises(ValueError):
        ma.multiply(M.DistributedVector.fromVector(None, x, 4))
    with pytest.raises(ValueError):
        ma.multiply(M.DistributedVector.fromVector(None, np.ones(5), 2))


@pytest.mark.parametrize("dims,grid", [((600, 600), (3, 2)), ((1000, 1000), (4, 4)), ((777, 777), (2, 3))])
def test_matrix_vector_vs_oracle(M, oracle, dims, grid):
    """BlockMatrix.multiply(DistributedVector) on random data against the oracle running the same algorithm
    (block x piece by F2J dgemv, ascending reduce)."""
    m, n = dims
    rng = np.random.default_rng(m + grid[0])
    A, x = rng.random((m, n)) * 2 - 1, rng.random(n) * 2 - 1
    rows = list(enumerate(A))
    ga = M.DenseVecMatrix(rows).toBlockMatrix(*grid)
    oa = oracle.DenseVecMatrix(rows).to_block_matrix(*grid)
    gv, ov = M.DistributedVector.fromVector(None, x, grid[1]), oracle.DistributedVector.from_vector(x, grid[1])
    got, ref = ga.multiply(gv), oa.multiply_dist_vector(ov)
    assert got.splitNum == ref.split_num() and got.length == ref.length()
    gp = {i: p.toBreeze().reshape(-1) for i, p in got.vectors}
    denom = np.abs(A) @ np.abs(x)
    bm = -(-m // grid[0])
    for i, piece in ref.vectors:
        assert (np.abs(gp[i] - piece) / denom[i * bm:i * bm + piece.shape[0]]).max() <= TOL
    # broadcast-vector overloads
    y = M.DenseVecMatrix(rows).multiply(x)
    assert (np.abs(y - oracle.DenseVecMatrix(rows).multiply_vector(x)) / denom).max() <= TOL
    y2 = M.DenseVecMatrix(rows).multiply(x, grid[0]).toBreeze()
    assert (np.abs(y2 - oracle.DenseVecMatrix(rows).multiply_vector(x, grid[0]).to_breeze()) / denom).max() <= TOL


def test_random_dist_vector_bit_exact(M, oracle):
    """MTUtils.randomDistVector: piece i = the first values of the stream of partition seed i (rdd/RandomRDD.scala:
    103-134), bit-identical to the oracle's XORShift restatement; onesDistVector."""
    v = M.MTUtils.randomDistVector(None, 1000, 3, seed=99)
    seeds = oracle.java_random_longs(99, 3)
    lens = [334, 334, 332]
    assert v.length == 1000 and v.splitNum == 3
    for (i, p), s, n in zip(sorted(v.vectors, key=lambda t: t[0]), seeds, lens):
        assert p.rows == n
        assert np.array_equal(p.toBreeze().reshape(-1), oracle.uniform_stream(s, 0, n))
    ones = M.MTUtils.onesDistVector(None, 10, 3)
    assert ones.length == 10 and np.array_equal(np.concatenate([p.toBreeze().reshape(-1) for _, p in ones.vectors]), np.ones(10))

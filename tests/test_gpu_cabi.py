"""GPU parity tests at the C-ABI boundary: every kernel against the CPU oracle on the same inputs.

Tolerances: element-wise / transpose / fill are BIT-EXACT (integer/byte-level work and single IEEE ops);
fp64 GEMM must satisfy  max_ij |C - C_ref|_ij / (|A||B|)_ij <= 1e-10  and  ||C - C_ref||_F / ||C_ref||_F <= 1e-10
(BASELINE.json north_star; SURVEY §8d) — in practice both are ~1e-16 * sqrt(K).
"""
import ctypes as C

import numpy as np
import pytest

from marlin_b200 import _native as nat
from tests.harness import gpu  # noqa: F401  (a fixture)

pytestmark = pytest.mark.gpu
TOL = 1e-10


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


def upload(gpu, arr, offset=0, rows=None, cols=None, ld=None, trans=0, dtype=nat.MB_F64):
    lib, ctx = gpu
    flat = np.ascontiguousarray(arr, dtype=np.float64).reshape(-1)
    h = nat.c_blk()
    nat.check(lib.mb_block_upload(ctx, _vp(flat), offset, rows, cols, ld, trans, dtype, C.byref(h)))
    return h


def upload_mat(gpu, mat, dtype=nat.MB_F64):
    f = np.asfortranarray(mat, dtype=np.float64)
    return upload(gpu, f.reshape(-1, order="F"), 0, f.shape[0], f.shape[1], max(1, f.shape[0]), 0, dtype)


def download(gpu, h, rows, cols):
    lib, ctx = gpu
    out = np.empty((rows, cols), order="F")
    nat.check(lib.mb_block_download(ctx, h, _vp(out), max(1, rows)))
    return out


def alloc(gpu, rows, cols, dtype=nat.MB_F64):
    lib, ctx = gpu
    h = nat.c_blk()
    nat.check(lib.mb_block_alloc(ctx, rows, cols, dtype, C.byref(h)))
    return h


def gemm_errors(got, ref, A, B):
    denom = np.abs(A) @ np.abs(B)
    denom[denom == 0] = 1.0
    return (np.abs(got - ref) / denom).max(), np.linalg.norm(got - ref) / max(np.linalg.norm(ref), 1e-300)


# ---------------------------------------------------------------------------------------- GEMM
def test_golden_4x4_product_exact(gpu):
    """DistributedMatrixSuite.scala:253-262: A*A for the suite's 4x4 matrix, exact."""
    from tests import marlin_cases as mc
    lib, ctx = gpu
    a = upload_mat(gpu, mc.EXPECTED_DENSE)
    c = alloc(gpu, 4, 4)
    nat.check(lib.mb_block_gemm(ctx, a, a, c, 0))
    assert np.array_equal(download(gpu, c, 4, 4), mc.EXPECTED_PRODUCT)
    nat.check(lib.mb_block_gemm(ctx, a, a, c, 1))            # accumulate: the reduceByKey add fused in
    assert np.array_equal(download(gpu, c, 4, 4), 2 * mc.EXPECTED_PRODUCT)


@pytest.mark.parametrize("shape", [(1, 1, 1), (2, 3, 5), (8, 8, 4), (50, 50, 50), (100, 100, 100), (127, 129, 17),
                                   (128, 128, 16), (130, 126, 50), (257, 383, 1000), (640, 512, 96)])
@pytest.mark.parametrize("ta", [0, 1])
@pytest.mark.parametrize("tb", [0, 1])
def test_block_gemm_vs_f2j_oracle(gpu, oracle, shape, ta, tb):
    """mb_block_gemm on Breeze-style views (isTranspose on either side) vs the F2J-order oracle."""
    lib, ctx = gpu
    m, n, k = shape
    rng = np.random.default_rng(m * 1000 + n * 10 + k + 2 * ta + tb)
    A = rng.random((m, k)) * 2 - 1
    B = rng.random((k, n)) * 2 - 1
    ref = oracle.block_multiply(np.ascontiguousarray(A) if ta else np.asfortranarray(A),
                                np.ascontiguousarray(B) if tb else np.asfortranarray(B), "f2j")
    # a transposed view = the column-major array of X^T with is_transpose=1
    ha = upload(gpu, np.asfortranarray(A.T).reshape(-1, order="F"), 0, m, k, max(1, k), 1) if ta else upload_mat(gpu, A)
    hb = upload(gpu, np.asfortranarray(B.T).reshape(-1, order="F"), 0, k, n, max(1, n), 1) if tb else upload_mat(gpu, B)
    hc = alloc(gpu, m, n)
    nat.check(lib.mb_block_gemm(ctx, ha, hb, hc, 0))
    got = download(gpu, hc, m, n)
    e_scaled, e_norm = gemm_errors(got, ref, A, B)
    assert e_scaled <= TOL and e_norm <= TOL, (e_scaled, e_norm)
    for h in (ha, hb, hc):
        lib.mb_block_free(ctx, h)


def test_views_transposed_without_copy(gpu, oracle):
    """is_transpose views built on device (mb_block_view_t) feed the 'T' kernels; row-major C via C^T = B^T A^T."""
    lib, ctx = gpu
    rng = np.random.default_rng(3)
    A, B = rng.random((96, 70)), rng.random((70, 44))
    hat = upload_mat(gpu, A.T)
    hbt = upload_mat(gpu, B.T)
    va, vb = nat.c_blk(), nat.c_blk()
    nat.check(lib.mb_block_view_t(ctx, hat, C.byref(va)))
    nat.check(lib.mb_block_view_t(ctx, hbt, C.byref(vb)))
    ref = A @ B
    hc = alloc(gpu, 96, 44)
    nat.check(lib.mb_block_gemm(ctx, va, vb, hc, 0))
    assert gemm_errors(download(gpu, hc, 96, 44), ref, A, B)[0] <= TOL
    # transposed (row-major) result block
    hct = alloc(gpu, 44, 96)
    vct = nat.c_blk()
    nat.check(lib.mb_block_view_t(ctx, hct, C.byref(vct)))
    nat.check(lib.mb_block_gemm(ctx, va, vb, vct, 0))
    assert gemm_errors(download(gpu, hct, 44, 96).T, ref, A, B)[0] <= TOL


def test_odd_ld_and_offset_falls_back_to_generic(gpu, oracle):
    """Views with odd majorStride / odd offset break TMA's 16-byte rule: the CUDA-core kernel must take over."""
    lib, ctx = gpu
    rng = np.random.default_rng(4)
    parent = rng.random((51, 37))
    hp = upload_mat(gpu, parent)                        # ld = 51 (odd)
    sl = nat.c_blk()
    nat.check(lib.mb_block_slice(ctx, hp, 3, 33, 1, 21, C.byref(sl)))     # 30 x 20 view at odd offset
    B = rng.random((20, 9))
    hb = upload_mat(gpu, B)
    hc = alloc(gpu, 30, 9)
    nat.check(lib.mb_block_gemm(ctx, sl, hb, hc, 0))
    A = parent[3:33, 1:21]
    ref = oracle.block_multiply(np.asfortranarray(A), np.asfortranarray(B), "f2j")
    assert gemm_errors(download(gpu, hc, 30, 9), ref, A, B)[0] <= TOL


def test_dgemm_host_netlib_signature(gpu, oracle):
    """mb_dgemm_host = netlib BLAS.dgemm with offsets / leading dims / alpha / beta on host arrays."""
    lib, ctx = gpu
    rng = np.random.default_rng(5)
    m, n, k, lda, ldb, ldc = 33, 29, 41, 40, 45, 37
    a = rng.random(7 + lda * k); b = rng.random(3 + ldb * n); c = rng.random(5 + ldc * n)
    ref = c.copy()
    oracle.dgemm_f2j("N", "N", m, n, k, 1.5, a, 7, lda, b, 3, ldb, -0.5, ref, 5, ldc)
    got = c.copy()
    nat.check(lib.mb_dgemm_host(ctx, b"N", b"N", m, n, k, 1.5, _vp(a), 7, lda, _vp(b), 3, ldb, -0.5, _vp(got), 5, ldc))
    assert np.allclose(got, ref, rtol=1e-12, atol=1e-12)
    pad = np.ones(len(c), bool)
    for j in range(n):
        pad[5 + j * ldc:5 + j * ldc + m] = False
    assert np.array_equal(got[pad], c[pad])             # padding between columns untouched
    # transposed operands
    a2 = rng.random(44 * m); b2 = rng.random(ldb * k)      # op(A) = A^T: A is k x m with leading dimension 44
    ref2 = np.zeros(ldc * n); got2 = np.zeros(ldc * n)
    oracle.dgemm_f2j("T", "T", m, n, k, 1.0, a2, 0, 44, b2, 0, 30, 0.0, ref2, 0, ldc)
    nat.check(lib.mb_dgemm_host(ctx, b"T", b"T", m, n, k, 1.0, _vp(a2), 0, 44, _vp(b2), 0, 30, 0.0, _vp(got2), 0, ldc))
    assert np.allclose(got2, ref2, rtol=1e-12, atol=1e-12)


def test_error_codes(gpu):
    lib, ctx = gpu
    a, b, c = alloc(gpu, 4, 3), alloc(gpu, 4, 4), alloc(gpu, 4, 4)
    assert lib.mb_block_gemm(ctx, a, b, c, 0) == nat.MB_ERR_DIM_MISMATCH
    assert b"Dimension mismatch during matrix-matrix multiplication: 3 vs 4" in lib.mb_last_error()   # BlockMatrix.scala:150-151
    assert lib.mb_block_add(ctx, a, b, c) == nat.MB_ERR_DIM_MISMATCH
    assert lib.mb_block_gemm(ctx, None, b, c, 0) == nat.MB_ERR_INVALID_ARG


@pytest.mark.parametrize("size", [1024, 4096])
def test_full_size_properties(gpu, size):
    """BASELINE config[1] size (4096^2, single block): size-independent checks —
    Freivalds (C x == A (B x) in fp64 on the host, O(n^2)), linearity under accumulate, and agreement of the
    tensor-core kernel with the independent CUDA-core kernel on a sampled sub-block."""
    import torch
    lib, ctx = gpu
    n = size
    g = torch.Generator(device="cuda").manual_seed(42)
    A = torch.rand(n, n, device="cuda", dtype=torch.float64, generator=g)      # storage (cols, rows) == column-major
    B = torch.rand(n, n, device="cuda", dtype=torch.float64, generator=g)
    Cm = torch.empty(n, n, device="cuda", dtype=torch.float64)
    torch.cuda.synchronize()
    p = lambda t: C.c_void_p(t.data_ptr())
    nat.check(lib.mb_dgemm_device(ctx, b"N", b"N", n, n, n, 1.0, p(A), n, p(B), n, 0.0, p(Cm), n))
    nat.check(lib.mb_synchronize(ctx))
    Ah, Bh, Ch = A.cpu().numpy().T, B.cpu().numpy().T, Cm.cpu().numpy().T          # logical matrices
    rng = np.random.default_rng(0)
    for _ in range(3):
        x = rng.random(n)
        lhs, rhs = Ch @ x, Ah @ (Bh @ x)
        assert np.abs(lhs - rhs).max() / np.abs(rhs).max() <= TOL
    # linearity: C += A*B twice more -> 3C
    nat.check(lib.mb_dgemm_device(ctx, b"N", b"N", n, n, n, 1.0, p(A), n, p(B), n, 1.0, p(Cm), n))
    nat.check(lib.mb_dgemm_device(ctx, b"N", b"N", n, n, n, 1.0, p(A), n, p(B), n, 1.0, p(Cm), n))
    nat.check(lib.mb_synchronize(ctx))
    assert np.abs(Cm.cpu().numpy().T - 3 * Ch).max() <= 1e-10 * np.abs(Ch).max()
    # independent kernel on a 256-column slab
    Cg = torch.empty(256, n, device="cuda", dtype=torch.float64)
    nat.check(lib.mb_dgemm_device_generic(ctx, b"N", b"N", n, 256, n, 1.0, p(A), n, p(B), n, 0.0, p(Cg), n))
    nat.check(lib.mb_synchronize(ctx))
    ref = Cg.cpu().numpy().T
    assert np.abs(Ch[:, :256] - ref).max() / np.abs(ref).max() <= 1e-12


# --------------------------------------------------------------------------- element-wise etc.
@pytest.mark.parametrize("shape", [(4, 4), (1, 7), (33, 17), (128, 64), (1000, 37), (512, 512)])
def test_elementwise_bit_exact(gpu, shape):
    lib, ctx = gpu
    rng = np.random.default_rng(shape[0] * 31 + shape[1])
    A = rng.random(shape) * 4 - 2
    B = rng.random(shape) * 4 - 2 + 0.1
    ha, hb, ho = upload_mat(gpu, A), upload_mat(gpu, B), alloc(gpu, *shape)
    for fn, ref in ((lib.mb_block_add, A + B), (lib.mb_block_sub, A - B), (lib.mb_block_hadamard, A * B)):
        nat.check(fn(ctx, ha, hb, ho))
        assert np.array_equal(download(gpu, ho, *shape), ref)
    for alpha, beta in ((1.0, 1.0), (2.0, 0.0), (-1.0, 3.25), (0.3, -0.7)):
        nat.check(lib.mb_block_axpb(ctx, ha, alpha, beta, ho))
        assert np.array_equal(download(gpu, ho, *shape), alpha * A + beta)      # two roundings, no FMA
    nat.check(lib.mb_block_div(ctx, hb, 3.0, 0, ho))
    assert np.array_equal(download(gpu, ho, *shape), B / 3.0)
    nat.check(lib.mb_block_div(ctx, hb, 3.0, 1, ho))
    assert np.array_equal(download(gpu, ho, *shape), 3.0 / B)


@pytest.mark.parametrize("shape", [(2, 2), (4, 2), (3, 5), (64, 64), (100, 36), (257, 129), (1024, 768), (2, 4096)])
def test_transpose_bit_exact(gpu, oracle, shape):
    lib, ctx = gpu
    A = np.random.default_rng(shape[0] + shape[1]).random(shape)
    ha, ho = upload_mat(gpu, A), alloc(gpu, shape[1], shape[0])
    nat.check(lib.mb_block_transpose(ctx, ha, ho))
    assert np.array_equal(download(gpu, ho, shape[1], shape[0]), oracle.block_transpose(A))
    # transposing a transposed view is a plain copy
    vt = nat.c_blk()
    nat.check(lib.mb_block_view_t(ctx, ha, C.byref(vt)))
    ho2 = alloc(gpu, *shape)
    nat.check(lib.mb_block_transpose(ctx, vt, ho2))
    assert np.array_equal(download(gpu, ho2, *shape), A)


def test_mixed_orientation_elementwise_and_slices(gpu):
    lib, ctx = gpu
    rng = np.random.default_rng(9)
    A, B = rng.random((40, 24)), rng.random((40, 24))
    ha = upload_mat(gpu, A)
    hbt = upload_mat(gpu, B.T)
    vb = nat.c_blk()
    nat.check(lib.mb_block_view_t(ctx, hbt, C.byref(vb)))            # logical 40x24, row-major storage
    ho = alloc(gpu, 40, 24)
    nat.check(lib.mb_block_add(ctx, ha, vb, ho))
    assert np.array_equal(download(gpu, ho, 40, 24), A + B)
    sa, sb, so = nat.c_blk(), nat.c_blk(), nat.c_blk()
    nat.check(lib.mb_block_slice(ctx, ha, 5, 25, 3, 13, C.byref(sa)))
    nat.check(lib.mb_block_slice(ctx, vb, 5, 25, 3, 13, C.byref(sb)))
    nat.check(lib.mb_block_slice(ctx, ho, 0, 20, 0, 10, C.byref(so)))
    nat.check(lib.mb_block_sub(ctx, sa, sb, so))
    got = download(gpu, ho, 40, 24)
    assert np.array_equal(got[:20, :10], A[5:25, 3:13] - B[5:25, 3:13])
    assert np.array_equal(got[20:, :], (A + B)[20:, :])             # rest of the parent untouched


def test_sum(gpu):
    lib, ctx = gpu
    from tests import marlin_cases as mc
    out = C.c_double()
    nat.check(lib.mb_block_sum(ctx, upload_mat(gpu, mc.EXPECTED_DENSE), C.byref(out)))
    assert out.value == mc.SUM                                       # DMS.scala:319-324
    A = np.random.default_rng(2).random((777, 333))
    nat.check(lib.mb_block_sum(ctx, upload_mat(gpu, A), C.byref(out)))
    assert out.value == pytest.approx(A.sum(), rel=1e-13)
    nat.check(lib.mb_block_sum(ctx, upload_mat(gpu, A), C.byref(out)))
    first = out.value
    nat.check(lib.mb_block_sum(ctx, upload_mat(gpu, A), C.byref(out)))
    assert out.value == first                                        # fixed reduction tree: reproducible


def test_upload_rounds_to_bf16_rne_and_back(gpu):
    lib, ctx = gpu
    import torch
    A = np.random.default_rng(8).random((37, 21))
    h = upload_mat(gpu, A, nat.MB_BF16)
    got = download(gpu, h, 37, 21)
    # direct RNE double->bf16 (NOT double->float->bf16): emulate with integer arithmetic on the fp64 bits
    bits = A.view(np.uint64)
    f32 = A.astype(np.float32)
    ref = torch.from_numpy(A).to(torch.bfloat16).to(torch.float64).numpy()
    # torch rounds via float32; the two differ only on exact double-rounding ties, so accept either but
    # require |got - A| <= half a bf16 ulp
    ulp = 2.0 ** (np.floor(np.log2(np.abs(A))) - 7)
    assert (np.abs(got - A) <= ulp / 2).all()
    assert (got == ref).mean() > 0.999


@pytest.mark.parametrize("row_major", [0, 1])
def test_fill_uniform_bit_exact_with_oracle_stream(gpu, oracle, row_major):
    """On-device XORShift jump-ahead generator == the sequential restatement of UniformGenerator.nextValue()."""
    lib, ctx = gpu
    rows, cols = 61, 47
    h = alloc(gpu, rows, cols)
    seed, first = 123456789, 1000
    nat.check(lib.mb_fill_uniform(ctx, h, seed, first, 0.0, 1.0, row_major))
    got = download(gpu, h, rows, cols)
    stream = oracle.uniform_stream(seed, first, rows * cols)
    ref = stream.reshape(rows, cols) if row_major else stream.reshape((rows, cols), order="F")
    assert np.array_equal(got, ref)
    nat.check(lib.mb_fill_uniform(ctx, h, -42, 0, -2.0, 5.0, row_major))
    stream = oracle.uniform_stream(-42, 0, rows * cols, -2.0, 5.0)
    ref = stream.reshape(rows, cols) if row_major else stream.reshape((rows, cols), order="F")
    assert np.array_equal(download(gpu, h, rows, cols), ref)


@pytest.mark.parametrize("row_major", [0, 1])
def test_fill_uniform_many_ctas_and_far_offsets(gpu, oracle, row_major):
    """Several CTAs with a ragged tail (every thread owns a long run and jumps to it), stream offsets beyond 2^33, and a
    strided destination (slice of a larger block) that takes the non-linear store path."""
    lib, ctx = gpu
    rows, cols = 701, 613                                   # 429,713 values: 6 full CTAs of 65,536 + a partial one
    h = alloc(gpu, rows, cols)
    for seed, first in ((2024, 0), (-7, (1 << 33) + 12345), (31, (1 << 38) - 3)):
        nat.check(lib.mb_fill_uniform(ctx, h, seed, first, 0.0, 1.0, row_major))
        stream = oracle.uniform_stream_far(seed, first, rows * cols)      # independent GF(2) matrix power, then sequential
        ref = stream.reshape(rows, cols) if row_major else stream.reshape((rows, cols), order="F")
        assert np.array_equal(download(gpu, h, rows, cols), ref)
    # a non-unit range on full CTAs (the fast kernel's affine path: two roundings, a + (b - a) * x as on the JVM)
    nat.check(lib.mb_fill_uniform(ctx, h, 77, 5, -2.0, 5.0, row_major))
    stream = oracle.uniform_stream(77, 5, rows * cols, -2.0, 5.0)
    ref = stream.reshape(rows, cols) if row_major else stream.reshape((rows, cols), order="F")
    assert np.array_equal(download(gpu, h, rows, cols), ref)
    big = alloc(gpu, rows + 9, cols + 5)
    nat.check(lib.mb_block_fill(ctx, big, -1.0))
    view = nat.c_blk()
    nat.check(lib.mb_block_slice(ctx, big, 4, 4 + rows, 2, 2 + cols, C.byref(view)))
    nat.check(lib.mb_fill_uniform(ctx, view, 99, 77, 0.0, 1.0, row_major))
    stream = oracle.uniform_stream(99, 77, rows * cols)
    ref = stream.reshape(rows, cols) if row_major else stream.reshape((rows, cols), order="F")
    full = download(gpu, big, rows + 9, cols + 5)
    assert np.array_equal(full[4:4 + rows, 2:2 + cols], ref)
    full[4:4 + rows, 2:2 + cols] = -1.0
    assert np.all(full == -1.0)                             # nothing written outside the view


def test_fill_uniform_fast_kernel_is_the_one_that_ran(gpu, oracle):
    """The bit-exactness assertions above hold for whichever generator kernel ran; this one shows WHICH: full CTAs of a
    packed block go to the fast kernel (IMAD.WIDE shifts + magic-number conversion) and only the ragged tail to the general
    one, i.e. two launches — unless the library's once-per-device self-check (fast kernel vs general kernel, on the device)
    has disabled the fast kernel, which would be a finding in its own right.  Runs after the other single-process tests
    (tests/conftest.py) so that such a finding cannot hide their results under -x."""
    lib, ctx = gpu
    rows, cols = 701, 613                                   # 6 full CTAs + a partial one
    h = alloc(gpu, rows, cols)
    l0 = lib.mb_launch_count(ctx)
    nat.check(lib.mb_fill_uniform(ctx, h, 5, 0, 0.0, 1.0, 0))
    assert lib.mb_launch_count(ctx) - l0 == 2, "fast generator kernel not active (disabled by its self-check)"
    assert np.array_equal(download(gpu, h, rows, cols), oracle.uniform_stream(5, 0, rows * cols).reshape((rows, cols), order="F"))
    exact = alloc(gpu, 512, 256)                            # exactly two full CTAs: no tail launch
    l0 = lib.mb_launch_count(ctx)
    nat.check(lib.mb_fill_uniform(ctx, exact, 6, 9, -1.0, 1.0, 0))
    assert lib.mb_launch_count(ctx) - l0 == 1
    assert np.array_equal(download(gpu, exact, 512, 256),
                          oracle.uniform_stream(6, 9, 512 * 256, -1.0, 1.0).reshape((512, 256), order="F"))


def test_matmul_blocked_seq_order(gpu, oracle):
    """mb_matmul_blocked == BlockMatrix.multiply (BlockMatrix.scala:149-186) for a ragged (3,2,2) grid."""
    lib, ctx = gpu
    rng = np.random.default_rng(11)
    M, K, N, m, k, n = 50, 37, 29, 3, 2, 2
    A, B = rng.random((M, K)), rng.random((K, N))
    oa = oracle.DenseVecMatrix(list(enumerate(A))).to_block_matrix(m, k)
    ob = oracle.DenseVecMatrix(list(enumerate(B))).to_block_matrix(k, n)
    ref = oa.multiply(ob, gemm="f2j")
    ta = {key: blk for key, blk in oa.blocks}
    tb = {key: blk for key, blk in ob.blocks}
    a_h = (nat.c_blk * (m * k))(*[upload_mat(gpu, ta[(i, kk)]) for i in range(m) for kk in range(k)])
    b_h = (nat.c_blk * (k * n))(*[upload_mat(gpu, tb[(kk, j)]) for kk in range(k) for j in range(n)])
    shapes = {(i, j): (ta[(i, 0)].shape[0], tb[(0, j)].shape[1]) for i in range(m) for j in range(n)}
    c_h = (nat.c_blk * (m * n))(*[alloc(gpu, *shapes[(i, j)]) for i in range(m) for j in range(n)])
    nat.check(lib.mb_matmul_blocked(ctx, a_h, b_h, m, k, n, c_h))
    refb = dict(ref.blocks)
    for i in range(m):
        for j in range(n):
            got = download(gpu, c_h[i * n + j], *shapes[(i, j)])
            assert np.abs(got - refb[(i, j)]).max() <= 1e-12


def upload_even_ld(gpu, mat):
    """A column-major device block whose leading dimension is even (TMA eligibility of the DMMA kernels: 16-byte
    rows), whatever the row count: odd-row matrices become a view [0:rows) of a (rows + 1)-row allocation."""
    lib, ctx = gpu
    rows, cols = mat.shape
    if rows % 2 == 0:
        return upload_mat(gpu, mat)
    big = alloc(gpu, rows + 1, cols)
    view = nat.c_blk()
    nat.check(lib.mb_block_slice(ctx, big, 0, rows, 0, cols, C.byref(view)))
    packed = upload_mat(gpu, mat)
    nat.check(lib.mb_block_copy(ctx, packed, view))
    nat.check(lib.mb_block_free(ctx, packed))
    return view


@pytest.mark.parametrize("dims", [(1000, 900, 1100, 2, 3, 2), (700, 530, 900, 2, 3, 2), (2048, 2048, 2048, 2, 2, 2),
                                  (1500, 260, 300, 3, 2, 1), (390, 4100, 650, 1, 4, 2)])
def test_matmul_blocked_grouped_kernel_multitile_ragged(gpu, oracle, dims):
    """The headline kernel, gemm_f64_dmma_grouped_kernel, against the oracle on blocks that span SEVERAL 128x128 CTA
    tiles, with ragged last blocks (ceil sizing, BlockMatrix.scala:73-74), ragged K segments and more than one C block
    per launch: tile location across C blocks (locate / tile_coords), banding, multi-wave scheduling and the K loop
    concatenated over kk.  Every tile gets an even leading dimension so the launch IS the grouped one — asserted through
    the launch counter (one launch for the whole multiply; the per-product fallback would need m*k*n)."""
    lib, ctx = gpu
    M, K, N, m, k, n = dims
    rng = np.random.default_rng(M + K + N)
    A, B = rng.random((M, K)) - 0.5, rng.random((K, N)) - 0.5
    oa = oracle.DenseVecMatrix(list(enumerate(A))).to_block_matrix(m, k)
    ob = oracle.DenseVecMatrix(list(enumerate(B))).to_block_matrix(k, n)
    ref = dict(oa.multiply(ob, gemm="blas" if M * K * N > 4e8 else "f2j").blocks)
    ta, tb = dict(oa.blocks), dict(ob.blocks)
    a_h = (nat.c_blk * (m * k))(*[upload_even_ld(gpu, ta[(i, kk)]) for i in range(m) for kk in range(k)])
    b_h = (nat.c_blk * (k * n))(*[upload_even_ld(gpu, tb[(kk, j)]) for kk in range(k) for j in range(n)])
    shapes = {(i, j): (ta[(i, 0)].shape[0], tb[(0, j)].shape[1]) for i in range(m) for j in range(n)}
    c_h = (nat.c_blk * (m * n))(*[alloc(gpu, *shapes[(i, j)]) for i in range(m) for j in range(n)])
    for c in c_h:
        nat.check(lib.mb_block_fill(ctx, c, float("nan")))          # the grouped launch overwrites, never accumulates
    l0 = lib.mb_launch_count(ctx)
    nat.check(lib.mb_matmul_blocked(ctx, a_h, b_h, m, k, n, c_h))
    assert lib.mb_launch_count(ctx) - l0 == 1, "expected ONE grouped launch"
    worst = 0.0
    for i in range(m):
        for j in range(n):
            got = download(gpu, c_h[i * n + j], *shapes[(i, j)])
            Ai = np.hstack([ta[(i, kk)] for kk in range(k)])
            Bj = np.vstack([tb[(kk, j)] for kk in range(k)])
            e1, e2 = gemm_errors(got, ref[(i, j)], Ai, Bj)
            assert e1 <= TOL and e2 <= TOL, (i, j, e1, e2)
            worst = max(worst, e1)
    # a subset call (two C blocks of the grid) is again one grouped launch and leaves the other blocks untouched
    if m * n >= 3:
        for c in c_h:
            nat.check(lib.mb_block_fill(ctx, c, -7.0))
        ids = (C.c_int32 * 2)(m * n - 1, 0)
        l0 = lib.mb_launch_count(ctx)
        nat.check(lib.mb_matmul_blocked_subset(ctx, a_h, b_h, m, k, n, c_h, ids, 2))
        assert lib.mb_launch_count(ctx) - l0 == 1
        for c in range(m * n):
            i, j = divmod(c, n)
            got = download(gpu, c_h[c], *shapes[(i, j)])
            if c in (0, m * n - 1):
                assert np.abs(got - ref[(i, j)]).max() <= 1e-11
            else:
                assert np.all(got == -7.0)


def test_matmul_blocked_full_size_freivalds(gpu):
    """8192^2 on a (2,2,2) grid through mb_matmul_blocked (ONE grouped launch, 4096 CTA tiles = 31 waves on 132 SMs, the
    same tile count per launch as one rank's share of the headline at 8 GPUs): Freivalds — C x == A (B x) with host fp64
    matvecs on the downloaded tiles, three random vectors, scaled error <= 1e-10 (U[0,1) inputs: |A||B| = A B)."""
    lib, ctx = gpu
    g, bs = 2, 4096
    n = g * bs
    tiles = {}
    for name, seed in (("A", 42), ("B", 43)):
        for r in range(g):
            for c in range(g):
                h = alloc(gpu, bs, bs)
                nat.check(lib.mb_fill_uniform(ctx, h, seed * 1000 + r * g + c, 0, 0.0, 1.0, 0))
                tiles[(name, r, c)] = h
    a_h = (nat.c_blk * (g * g))(*[tiles[("A", i, kk)] for i in range(g) for kk in range(g)])
    b_h = (nat.c_blk * (g * g))(*[tiles[("B", kk, j)] for kk in range(g) for j in range(g)])
    c_h = (nat.c_blk * (g * g))(*[alloc(gpu, bs, bs) for _ in range(g * g)])
    l0 = lib.mb_launch_count(ctx)
    nat.check(lib.mb_matmul_blocked(ctx, a_h, b_h, g, g, g, c_h))
    assert lib.mb_launch_count(ctx) - l0 == 1
    full = lambda hs: np.block([[download(gpu, hs[r * g + c], bs, bs) for c in range(g)] for r in range(g)])
    Ah, Bh, Ch = full(a_h), full(b_h), full(c_h)
    rng = np.random.default_rng(5)
    for _ in range(3):
        x = rng.random(n)
        lhs, rhs = Ch @ x, Ah @ (Bh @ x)
        assert (np.abs(lhs - rhs) / rhs).max() <= TOL
    for h in list(a_h) + list(b_h) + list(c_h):
        nat.check(lib.mb_block_free(ctx, h))


@pytest.mark.parametrize("dims", [(75, 64, 51, 2, 3, 2), (300, 200, 2100, 1, 2, 2), (260, 130, 1100, 1, 1, 1),
                                  (200, 2300, 260, 1, 2, 2), (131, 2111, 77, 2, 2, 1), (140, 1200, 1300, 2, 1, 2)])
def test_matmul_blocked_host_pipelined(gpu, oracle, dims):
    """mb_matmul_blocked_host: host tiles in, host tiles out (pipelined H2D / DMMA / D2H) == BlockMatrix.multiply.
    Column counts >= 1024 exercise the chunked last download (and, for a single product, the column-chunked upload of
    B); K extents >= 1024 exercise the K-chunked first product (quarters of A and B uploaded and multiplied in turn)."""
    lib, ctx = gpu
    rng = np.random.default_rng(12)
    M, K, N, m, k, n = dims
    A, B = rng.random((M, K)) - 0.5, rng.random((K, N)) - 0.5
    oa = oracle.DenseVecMatrix(list(enumerate(A))).to_block_matrix(m, k)
    ob = oracle.DenseVecMatrix(list(enumerate(B))).to_block_matrix(k, n)
    ref = dict(oa.multiply(ob, gemm="blas" if N > 1000 else "f2j").blocks)
    ta, tb = dict(oa.blocks), dict(ob.blocks)
    a_arr = [np.asfortranarray(ta[(i, kk)]) for i in range(m) for kk in range(k)]
    b_arr = [np.asfortranarray(tb[(kk, j)]) for kk in range(k) for j in range(n)]
    row_len = (C.c_int32 * m)(*[ta[(i, 0)].shape[0] for i in range(m)])
    k_len = (C.c_int32 * k)(*[ta[(0, kk)].shape[1] for kk in range(k)])
    col_len = (C.c_int32 * n)(*[tb[(0, j)].shape[1] for j in range(n)])
    c_arr = [np.full((row_len[i], col_len[j]), np.nan, order="F") for i in range(m) for j in range(n)]
    pa = (C.c_void_p * (m * k))(*[x.ctypes.data for x in a_arr])
    pb = (C.c_void_p * (k * n))(*[x.ctypes.data for x in b_arr])
    pc = (C.c_void_p * (m * n))(*[x.ctypes.data for x in c_arr])
    for _ in range(2):                       # second call reuses the workspace
        nat.check(lib.mb_matmul_blocked_host(ctx, pa, pb, m, k, n, row_len, k_len, col_len, pc))
        for i in range(m):
            for j in range(n):
                assert np.abs(c_arr[i * n + j] - ref[(i, j)]).max() <= 1e-12


@pytest.mark.parametrize("dims", [(1000, 1024, 96), (777, 130, 1030), (5, 3, 2), (300, 64, 1), (129, 0, 7)])
def test_matmul_rowsharded_host_pipelined(gpu, oracle, dims, monkeypatch):
    """mb_matmul_rowsharded_host: row-major rows in, row-major rows out (DenseVecMatrix.multiply(B: BDM) for JVM-held
    rows), many chunks through the three-slot ring (the chunk size is forced down to 1 MiB), and the device-resident
    twin mb_matmul_rowsharded on transposed views."""
    lib, ctx = gpu
    monkeypatch.setenv("MARLIN_B200_ROWSHARD_CHUNK_MIB", "1")
    rows, k, n = dims
    rng = np.random.default_rng(rows + k)
    A = np.ascontiguousarray(rng.random((rows, k)) - 0.5)            # row-major rows
    B = np.asfortranarray(rng.random((k, n)) - 0.5)
    Cm = np.full((rows, n), np.nan)
    ref = A @ B
    denom = np.abs(A) @ np.abs(B)
    denom[denom == 0] = 1.0
    for _ in range(2):
        nat.check(lib.mb_matmul_rowsharded_host(ctx, _vp(A), rows, k, _vp(B), n, _vp(Cm)))
        assert (np.abs(Cm - ref) / denom).max() <= TOL
    if k > 0:
        ha = upload(gpu, A.reshape(-1), 0, rows, k, max(1, k), 1)
        hb = upload_mat(gpu, B)
        hct = alloc(gpu, n, rows)
        vct = nat.c_blk()
        nat.check(lib.mb_block_view_t(ctx, hct, C.byref(vct)))
        nat.check(lib.mb_matmul_rowsharded(ctx, ha, hb, vct))
        assert (np.abs(download(gpu, hct, n, rows).T - ref) / denom).max() <= TOL
        if k != n:
            assert lib.mb_matmul_rowsharded(ctx, hb, hb, vct) == nat.MB_ERR_DIM_MISMATCH


def test_dgemm_degenerate_cases(gpu):
    """netlib dgemm corner cases: k = 0 and alpha = 0 reduce to C := beta*C (dgemm.f quick returns), m or n = 0 is a no-op,
    bad arguments are rejected like xerbla."""
    import torch
    lib, ctx = gpu
    p = lambda t: C.c_void_p(t.data_ptr())
    Cm = torch.arange(12, dtype=torch.float64, device="cuda").reshape(3, 4).contiguous()      # column-major 4 x 3
    A = torch.ones(8, dtype=torch.float64, device="cuda")
    ref = Cm.clone()
    nat.check(lib.mb_dgemm_device(ctx, b"N", b"N", 4, 3, 0, 1.0, p(A), 4, p(A), 1, 2.0, p(Cm), 4))
    nat.check(lib.mb_synchronize(ctx))
    assert torch.equal(Cm, 2.0 * ref)
    nat.check(lib.mb_dgemm_device(ctx, b"N", b"N", 4, 3, 2, 0.0, p(A), 4, p(A), 2, 0.0, p(Cm), 4))
    nat.check(lib.mb_synchronize(ctx))
    assert torch.equal(Cm, torch.zeros_like(Cm))
    assert lib.mb_dgemm_device(ctx, b"N", b"N", 0, 3, 2, 1.0, p(A), 1, p(A), 2, 0.0, p(Cm), 1) == nat.MB_OK
    assert lib.mb_dgemm_device(ctx, b"X", b"N", 4, 3, 2, 1.0, p(A), 4, p(A), 2, 0.0, p(Cm), 4) == nat.MB_ERR_INVALID_ARG
    assert lib.mb_dgemm_device(ctx, b"N", b"N", 4, 3, 2, 1.0, p(A), 3, p(A), 2, 0.0, p(Cm), 4) == nat.MB_ERR_INVALID_ARG   # lda < m
    assert lib.mb_dgemm_device(ctx, b"N", b"N", -1, 3, 2, 1.0, p(A), 4, p(A), 2, 0.0, p(Cm), 4) == nat.MB_ERR_INVALID_ARG


def test_threads_share_blocks(gpu, oracle):
    """Spark local[N] runs tasks as threads of one JVM (LocalSparkContext.scala:11): (i) threads with one context EACH
    run concurrently on shared block handles; (ii) threads sharing ONE context serialise on its lock where the context's
    scratch is used (sum, dot, gemv) and still get the right answers."""
    import threading
    lib, ctx = gpu
    rng = np.random.default_rng(77)
    A, B = rng.random((300, 200)) - 0.5, rng.random((200, 260)) - 0.5
    x = rng.random(200)
    ha, hb, hx = upload_mat(gpu, A), upload_mat(gpu, B), upload_mat(gpu, x.reshape(-1, 1))
    ref_c, ref_y, ref_s = A @ B, A @ x, float(A.sum())
    errors = []

    def work(own_ctx):
        try:
            c = ctx
            if own_ctx:
                c = nat.c_ctx()
                nat.check(lib.mb_init(0, C.byref(c)))
            for _ in range(20):
                hc, hy = nat.c_blk(), nat.c_blk()
                nat.check(lib.mb_block_alloc(c, 300, 260, nat.MB_F64, C.byref(hc)))
                nat.check(lib.mb_block_alloc(c, 300, 1, nat.MB_F64, C.byref(hy)))
                nat.check(lib.mb_block_gemm(c, ha, hb, hc, 0))
                nat.check(lib.mb_block_gemv(c, ha, hx, hy, 0))
                s = C.c_double()
                nat.check(lib.mb_block_sum(c, ha, C.byref(s)))
                got_c = np.empty((300, 260), order="F"); got_y = np.empty((300, 1), order="F")
                nat.check(lib.mb_block_download(c, hc, _vp(got_c), 300))
                nat.check(lib.mb_block_download(c, hy, _vp(got_y), 300))
                assert np.abs(got_c - ref_c).max() <= 1e-12 and np.abs(got_y[:, 0] - ref_y).max() <= 1e-12
                assert abs(s.value - ref_s) <= 1e-10
                lib.mb_block_free(c, hc); lib.mb_block_free(c, hy)
            if own_ctx:
                lib.mb_shutdown(c)
        except Exception as exc:                      # surfaced in the main thread
            errors.append(repr(exc))

    for own in (True, False):
        threads = [threading.Thread(target=work, args=(own,)) for _ in range(4)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        assert not errors, errors

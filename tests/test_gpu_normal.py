"""StandardNormalGenerator on the GPU (mb_fill_normal, mb_fill_spvec_normal and the MTUtils generators) bit for bit
against tests/normal_oracle.py: sizes around the tile and budget bounds and a multi-wave size, both fill orders on packed,
sliced and transposed views with a sentinel around them, seeds, (mean, variance) edge cases, positions_out, a first
budget that falls short, fdlibm branch coverage, run-to-run bits, errors, temporaries; the Python generators partition by
partition; and two gloo ranks against one."""
import ctypes as C
import os
import socket
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from marlin_b200 import _native as nat
from tests import normal_oracle as no

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
TILE = 32768                                              # MB_NORMAL_TILE_ATTEMPTS
EXPECTED_PAIRS = int(TILE * np.pi / 4)                    # a tile's expected accepted attempts: 25735


@pytest.fixture(scope="module")
def M():
    import marlin_b200 as mb
    mb.Runtime.get().sync_stream()
    return mb


@pytest.fixture(scope="module")
def gpu(M):
    rt = M.Runtime.get()
    return rt.lib, rt.ctx


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


def alloc(gpu, rows, cols, dtype=nat.MB_F64):
    lib, ctx = gpu
    h = nat.c_blk()
    nat.check(lib.mb_block_alloc(ctx, rows, cols, dtype, C.byref(h)))
    return h


def download(gpu, h, rows, cols):
    lib, ctx = gpu
    out = np.empty((rows, cols), order="F")
    nat.check(lib.mb_block_download(ctx, h, _vp(out), max(1, rows)))
    return out


def fill(gpu, h, seed, mean=0.0, variance=1.0, row_major=0):
    lib, ctx = gpu
    pos = C.c_int64(-1)
    nat.check(lib.mb_fill_normal(ctx, h, seed, mean, variance, row_major, C.byref(pos)))
    return pos.value


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def same(got, want):
    assert got.shape == want.shape
    eq = bits(got) == bits(want)
    assert eq.all(), f"{(~eq).sum()} of {eq.size} differ, first at {np.argwhere(~eq)[0]}"


def in_order(stream, rows, cols, row_major):
    return stream.reshape(rows, cols) if row_major else stream.reshape((rows, cols), order="F")


# ------------------------------------------------------------------------------------------------------ sizes and seeds
@pytest.mark.parametrize("n", [1, 2, 3, 5, 127, 2 * EXPECTED_PAIRS - 2, 2 * EXPECTED_PAIRS - 1, 2 * EXPECTED_PAIRS,
                               2 * EXPECTED_PAIRS + 1, 2 * EXPECTED_PAIRS + 2, 2 * EXPECTED_PAIRS + 3, 400_001])
@pytest.mark.parametrize("seed", [0, -77, 2 ** 40 + 3])
def test_sizes_bit_exact(gpu, oracle, n, seed):
    h = alloc(gpu, n, 1)
    pos = fill(gpu, h, seed)
    want, want_pos, _ = no.normal_stream(seed, n)
    same(download(gpu, h, n, 1)[:, 0], want)
    assert pos == want_pos


def test_multi_wave_size_reaches_every_branch(gpu, oracle):
    """33.6 million values (about 1000 tiles of 256 threads, several waves on 132 SMs), one stream across 4099 rows; the
    values reach every fdlibm branch but f == 0, which needs s to be exactly a power of two (one attempt in about 2^52)."""
    rows, cols = 4099, 8192
    lib, ctx = gpu
    h = nat.c_blk()
    nat.check(lib.mb_block_view_t(ctx, alloc(gpu, cols, rows), C.byref(h)))     # a row shard: rows back to back
    pos = fill(gpu, h, 987654321, row_major=1)
    got = download(gpu, h, rows, cols)
    want, want_pos, counts = no.normal_stream(987654321, rows * cols)
    same(got, in_order(want, rows, cols, 1))
    assert pos == want_pos
    assert all(counts.get(b, 0) > 0 for b in no.BRANCHES if b != "small_f0"), counts
    fill(gpu, h, 987654321, row_major=1)                  # a second call: the same bits
    same(download(gpu, h, rows, cols), got)


@pytest.mark.parametrize("mean,variance", [(0.0, 1.0), (3.5, 0.25), (-1e300, 4.0), (-0.0, 0.0), (float("inf"), 1.0)])
@pytest.mark.parametrize("row_major", [0, 1])
def test_mean_and_variance(gpu, oracle, mean, variance, row_major):
    rows, cols = 301, 77
    h = alloc(gpu, rows, cols)
    fill(gpu, h, 5, mean, variance, row_major)
    want, _, _ = no.normal_stream(5, rows * cols, mean, variance)
    got = download(gpu, h, rows, cols)
    same(got, in_order(want, rows, cols, row_major))      # signed zeros by their bits
    if variance == 0.0:
        assert np.signbit(got).any() and (~np.signbit(got)).any()


@pytest.mark.parametrize("variance", [-1.0, float("nan"), -0.0])
def test_negative_and_nan_variance(gpu, oracle, variance):
    h = alloc(gpu, 999, 3)
    fill(gpu, h, 8, 2.0, variance)
    got = download(gpu, h, 999, 3)
    if variance == 0.0:                                   # sqrt(-0.0) = -0.0: mean + (-0.0 * g)
        same(got, in_order(no.normal_stream(8, 999 * 3, 2.0, -0.0)[0], 999, 3, 0))
    else:
        assert np.isnan(got).all()


# ---------------------------------------------------------------------------------------------------------------- views
@pytest.mark.parametrize("row_major", [0, 1])
@pytest.mark.parametrize("kind", ["packed", "slice", "transposed"])
def test_views_and_nothing_outside(gpu, oracle, row_major, kind):
    lib, ctx = gpu
    rows, cols = 2345, 61
    pr, pc = rows + 7, cols + 5
    parent = alloc(gpu, pc, pr) if kind == "transposed" else alloc(gpu, pr, pc)
    nat.check(lib.mb_block_fill(ctx, parent, -123.0))
    v, r0, c0 = nat.c_blk(), 0, 0
    if kind == "packed":
        v, rows, cols = parent, pr, pc
    elif kind == "slice":
        r0, c0 = 3, 2
        nat.check(lib.mb_block_slice(ctx, parent, r0, r0 + rows, c0, c0 + cols, C.byref(v)))
    else:
        r0, c0 = 4, 1
        t = nat.c_blk()
        nat.check(lib.mb_block_view_t(ctx, parent, C.byref(t)))                  # pr x pc, row-major storage
        nat.check(lib.mb_block_slice(ctx, t, r0, r0 + rows, c0, c0 + cols, C.byref(v)))
    fill(gpu, v, -3, 1.0, 2.0, row_major)
    want = in_order(no.normal_stream(-3, rows * cols, 1.0, 2.0)[0], rows, cols, row_major)
    same(download(gpu, v, rows, cols), want)
    full = download(gpu, parent, pc, pr).T if kind == "transposed" else download(gpu, parent, pr, pc)
    full[r0:r0 + rows, c0:c0 + cols] = -123.0
    assert np.all(full == -123.0)                          # nothing written outside the view


@pytest.mark.parametrize("row_major", [0, 1])
def test_linear_view_off_a_16_byte_boundary(M, gpu, oracle, row_major):
    """A packed view starting 8 bytes past a 16-byte boundary (the store path without 16-byte stores)."""
    import torch
    lib, ctx = gpu
    rows, cols = 1001, 333
    buf = torch.full((rows * cols + 2,), -7.0, dtype=torch.float64, device=M.Runtime.get().device)
    v = nat.c_blk()
    ld = cols if row_major else rows
    nat.check(lib.mb_block_wrap(ctx, C.c_void_p(buf.data_ptr()), 1, rows, cols, ld, row_major, nat.MB_F64, C.byref(v)))
    fill(gpu, v, 99, 0.0, 1.0, row_major)
    nat.check(lib.mb_synchronize(ctx))
    host = buf.cpu().numpy()
    same(host[1:-1], no.normal_stream(99, rows * cols)[0])
    assert host[0] == -7.0 and host[-1] == -7.0
    nat.check(lib.mb_block_free(ctx, v))


# ------------------------------------------------------------------------------------------- budget, launches, errors
def test_first_budget_short_takes_an_extra_round(gpu, oracle):
    """pairs = 25735: the budget rule gives one tile (ceil(25735 * 4 / pi) = 32768 attempts); a seed whose first tile
    accepts fewer than 25735 attempts needs a second round, which is two more launches."""
    lib, ctx = gpu
    n = 2 * 25735
    assert no.budget_tiles(25735, TILE) == 1
    short = next(s for s in range(1000) if no.accepted_attempts(s, TILE).sum() < 25735)
    enough = next(s for s in range(1000) if no.accepted_attempts(s, TILE).sum() >= 25735)
    assert no.counting_rounds(short, n, TILE) == 2 and no.counting_rounds(enough, n, TILE) == 1
    h = alloc(gpu, n, 1)
    for seed, launches in ((short, 5), (enough, 3)):
        l0 = lib.mb_launch_count(ctx)
        pos = fill(gpu, h, seed)
        assert lib.mb_launch_count(ctx) - l0 == launches
        want, want_pos, _ = no.normal_stream(seed, n)
        same(download(gpu, h, n, 1)[:, 0], want)
        assert pos == want_pos > 2 * TILE * (launches == 5)


def test_errors(gpu):
    lib, ctx = gpu
    bf = alloc(gpu, 4, 4, nat.MB_BF16)
    assert lib.mb_fill_normal(ctx, bf, 1, 0.0, 1.0, 0, None) == nat.MB_ERR_UNSUPPORTED
    assert "fp64" in lib.mb_last_error().decode()
    assert lib.mb_fill_normal(ctx, None, 1, 0.0, 1.0, 0, None) == nat.MB_ERR_INVALID_ARG
    assert lib.mb_fill_normal(None, alloc(gpu, 2, 2), 1, 0.0, 1.0, 0, None) != nat.MB_OK
    assert lib.mb_fill_spvec_normal(ctx, None, 1, 0.0, 1.0) == nat.MB_ERR_INVALID_ARG
    empty = alloc(gpu, 0, 5)
    pos = C.c_int64(-1)
    nat.check(lib.mb_fill_normal(ctx, empty, 1, 0.0, 1.0, 0, C.byref(pos)))
    assert pos.value == 0


def test_nothing_left_allocated(gpu):
    from tests.test_gpu_temporaries import _Pool
    lib, ctx = gpu
    pool = _Pool()
    h = alloc(gpu, 1000, 1000)
    fill(gpu, h, 4)
    nat.check(lib.mb_synchronize(ctx))
    before = pool.used()
    pool.reset_high()
    fill(gpu, h, 4)
    nat.check(lib.mb_synchronize(ctx))
    assert pool.high() > before and pool.used() == before
    nat.check(lib.mb_block_free(ctx, h))


# ---------------------------------------------------------------------------------------------------------- Python API
def _seeds(seed, n):
    from oracle import reference_model as rm
    return rm.java_random_longs(seed, n)


def test_random_den_vec_matrix(M, oracle):
    from marlin_b200.utils.mt_utils import StandardNormalGenerator
    nr, nc, P, seed = 61, 29, 5, 21
    got = M.MTUtils.randomDenVecMatrix(None, nr, nc, numPartitions=P, distribution=StandardNormalGenerator(-1.5, 2.25),
                                       seed=seed).toBreeze()
    seeds = _seeds(seed, P)
    for p in range(P):
        a, b = p * nr // P, (p + 1) * nr // P
        same(got[a:b], no.normal_stream(seeds[p], (b - a) * nc, -1.5, 2.25)[0].reshape(b - a, nc))


@pytest.mark.parametrize("dtype", [nat.MB_F64, nat.MB_F32])
def test_random_block_matrix(M, oracle, dtype):
    from marlin_b200.utils.mt_utils import StandardNormalGenerator
    nr, nc, br, bc, seed = 50, 37, 3, 4, 22
    bm = M.MTUtils.randomBlockMatrix(None, nr, nc, br, bc, distribution=StandardNormalGenerator(), seed=seed, dtype=dtype)
    brs, bcs = 17, 10                                     # ceil(50 / 3), ceil(37 / 4): the last row and column are ragged
    seeds = _seeds(seed, br * bc)
    want = np.zeros((nr, nc))
    for idx in range(br * bc):
        i, j = divmod(idx, bc)
        rows, cols = min(brs, nr - i * brs), min(bcs, nc - j * bcs)
        blk = no.normal_stream(seeds[idx], rows * cols)[0].reshape((rows, cols), order="F")
        want[i * brs:i * brs + rows, j * bcs:j * bcs + cols] = blk if dtype == nat.MB_F64 else blk.astype(np.float32)
    same(bm.toBreeze(), want)


def test_random_dist_vector(M, oracle):
    from marlin_b200.utils.mt_utils import StandardNormalGenerator
    v = M.MTUtils.randomDistVector(None, 101, 4, distribution=StandardNormalGenerator(0.5, 9.0), seed=24)
    seeds = _seeds(24, 4)
    pieces = dict(v.vectors)
    assert sorted(pieces) == [0, 1, 2, 3]
    for i, n in enumerate((26, 26, 26, 23)):             # split length ceil(101 / 4), the last piece the rest
        same(pieces[i].toBreeze()[:, 0], no.normal_stream(seeds[i], n, 0.5, 9.0)[0])


def test_random_spa_vec_matrix_draws_columns_after_the_values(M, oracle):
    from marlin_b200.utils.mt_utils import StandardNormalGenerator
    from oracle import reference_model as rm
    from tests import spvec_oracle as sv
    nr, nc, density, P, seed = 57, 40, 0.2, 5, 23
    sp = M.MTUtils.randomSpaVecMatrix(None, nr, nc, density, numPartitions=P, distribution=StandardNormalGenerator(-1.5, 2.25),
                                      seed=seed)
    s = int(nc * density)
    rp, ci, va = sp.block.to_host()
    assert np.array_equal(rp, np.arange(nr + 1) * s)
    seeds = _seeds(seed, P)
    for p in range(P):
        a, b = p * nr // P, (p + 1) * nr // P
        vals, positions, _ = no.normal_stream(seeds[p], s * (b - a), -1.5, 2.25)
        same(va[a * s:b * s], vals)
        cols = sv.column_set(rm.hash_seed(seeds[p]), positions, nc, s)       # positions [2A, 2A + nColumns)
        assert np.array_equal(ci[a * s:b * s].reshape(b - a, s), np.tile(cols, (b - a, 1)))


def test_zeros_and_ones_in_the_dense_generators(M):
    from marlin_b200.utils.mt_utils import OnesGenerator, ZerosGenerator
    for gen, value in ((ZerosGenerator(), 0.0), (OnesGenerator(), 1.0)):
        pieces = [p.toBreeze() for _, p in M.MTUtils.randomDistVector(None, 13, 3, distribution=gen, seed=1).vectors]
        assert [p.shape[0] for p in pieces] == [5, 5, 3]
        for got in [M.MTUtils.randomDenVecMatrix(None, 13, 7, distribution=gen, seed=1).toBreeze(),
                    M.MTUtils.randomBlockMatrix(None, 13, 7, 2, 3, distribution=gen, seed=1).toBreeze()] + pieces:
            same(got, np.full(got.shape, value))


def test_rejected_generators_name_themselves(M):
    from marlin_b200.utils.mt_utils import OnesGenerator, PoissonGenerator, ZerosGenerator

    def raises(call, name):
        with pytest.raises(M.MarlinArgumentError) as e:
            call()
        assert e.value.code == nat.MB_ERR_UNSUPPORTED and name in str(e.value), str(e.value)

    for gen in (PoissonGenerator(3.0), object()):
        name = "PoissonGenerator" if isinstance(gen, PoissonGenerator) else "unsupported distribution object"
        raises(lambda: M.MTUtils.randomDenVecMatrix(None, 5, 5, distribution=gen, seed=1), name)
        raises(lambda: M.MTUtils.randomBlockMatrix(None, 5, 5, 2, 2, distribution=gen, seed=1), name)
        raises(lambda: M.MTUtils.randomDistVector(None, 5, 2, distribution=gen, seed=1), name)
        raises(lambda: M.MTUtils.randomSpaVecMatrix(None, 5, 5, 0.5, distribution=gen, seed=1), name)
    for gen in (ZerosGenerator(), OnesGenerator()):
        raises(lambda: M.MTUtils.randomSpaVecMatrix(None, 5, 5, 0.5, distribution=gen, seed=1), type(gen).__name__)


# ---------------------------------------------------------------------------------------------------------- two ranks
def test_two_ranks_match_one(M, oracle, tmp_path):
    sys.path.insert(0, str(ROOT / "tests"))
    import normal_gpu_worker as w
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    env = dict(os.environ, NORMAL_WORKER_OUT=str(tmp_path / "r"))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), str(ROOT / "tests" / "normal_gpu_worker.py")]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900, env=env)
    assert out.returncode == 0, out.stdout[-4000:]
    for r in range(2):
        assert f"rank {r} normal generators ok" in out.stdout
    two = dict(np.load(str(tmp_path / "r.0.npz")))
    one = w.run(M)
    assert set(two) == set(one) - {"vector_1", "vector_3"}     # rank 0 holds pieces 0 and 2 of the vector
    for k in two:
        same(two[k], one[k])

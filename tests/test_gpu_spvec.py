"""SparseVecMatrix on the GPU: multiplySparse bit for bit against the oracle's fixed-order float32 sums
(tests/spvec_oracle.py) with rows on both sides of every bin bound, special values, empty rows, run-to-run and two-rank
determinism; toDenseVecMatrix, toSparseVecMatrix, randomSpaVecMatrix; the errors; and the chain into CoordinateMatrix."""
import math
import os
import socket
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from tests import spvec_oracle as sv

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]


def _mat(rows, n_rows, n_cols):
    import marlin_b200 as mb
    from marlin_b200.matrix.sparse_matrix import SparseVector
    return mb.SparseVecMatrix([(i, SparseVector(n_cols, ix, v)) for i, ix, v in rows], n_rows, n_cols)


def _coo(cm):
    order = np.lexsort((cm.cols, cm.rows))
    return cm.rows[order], cm.cols[order], cm.values[order]


def _assert_bits(got, want):
    gr, gc, gv = got
    wr, wc, wv = want
    assert np.array_equal(gr, wr) and np.array_equal(gc, wc)
    nan = np.isnan(wv)
    assert np.array_equal(np.isnan(gv), nan)                  # NaN payloads differ between the CPU and the GPU
    assert np.array_equal(gv[~nan].view(np.uint32), wv[~nan].view(np.uint32))


def _bin_case(seed=0):
    """B: rows 0..4999 with one entry, 5000..5999 with 64 (half of them inside 200 columns, so sums pile up), 6000..6099
    empty; n = 40000 columns, so wide rows span several windows.  A: one row per product count, on both sides of each
    bin bound, a row far beyond the CTA hash, an empty row and a row whose k all hit empty B rows."""
    from marlin_b200 import _native as nat
    rng = np.random.default_rng(seed)
    n, K = 40000, 6100
    B = []
    for k in range(K):
        if k < 5000:
            ix = rng.integers(0, n, 1)
        elif k < 6000:
            ix = np.sort(rng.choice(200 if k % 2 else n, 64, replace=False))
        else:
            continue
        B.append((k, ix, rng.standard_normal(ix.size) * 10.0 ** rng.integers(-3, 4, ix.size)))
    w, c = nat.MB_SPVEC_WARP_BOUND, nat.MB_SPVEC_CTA_BOUND
    targets = [1, 2, 63, w - 1, w, w + 1, c - 1, c, c + 1, 20000, 64000]
    A = []
    for i, u in enumerate(targets):
        longs = min(u // 64, 1000)
        singles = u - 64 * longs
        ks = np.sort(np.concatenate([rng.choice(1000, longs, replace=False) + 5000, rng.choice(5000, singles, replace=False)]))
        A.append((i, ks, rng.standard_normal(ks.size)))
    A.append((len(targets), np.zeros(0, np.int64), np.zeros(0)))
    A.append((len(targets) + 1, np.arange(6000, 6010), np.ones(10)))
    return A, B, len(A), K, n


def test_suite_sparse_matrix_multiply():
    """DistributedMatrixSuite.scala:152-162."""
    m = _mat(sv.SUITE_ROWS, 4, 4)
    assert np.array_equal(m.multiplySparse(_mat(sv.SUITE_ROWS, 4, 4)).toBreeze(), sv.SUITE_PRODUCT)


def test_suite_generate_random_sparse_matrix():
    """DistributedMatrixSuite.scala:147-150."""
    import marlin_b200 as mb
    s = mb.MTUtils.randomSpaVecMatrix(None, 10, 8, 0.3)
    assert s.nRows == 10 and s.elementsCount() == 10


def test_bins_bit_for_bit_and_run_to_run():
    A, B, m, K, n = _bin_case()
    want = sv.multiply_sparse(A, B)
    a, b = _mat(A, m, K), _mat(B, K, n)
    first = _coo(a.multiplySparse(b))
    _assert_bits(first, want)
    again = _coo(a.multiplySparse(b))
    assert all(np.array_equal(x, y) for x, y in zip(first[:2], again[:2]))
    assert np.array_equal(first[2].view(np.uint32), again[2].view(np.uint32))


def test_special_values():
    f32 = np.float32
    sub = float(f32(1e-40))                                   # a float32 subnormal
    A = [(0, [0, 1, 2, 3, 4, 5], [1.0, -1.0, -0.0, math.inf, 1e-20, 3.5e38]),
         (1, [0], [0.0]),
         (2, [6], [math.nan])]
    B = [(0, [0, 1, 2], [2.0, 0.0, sub]), (1, [0, 3], [2.0, 1.0]), (2, [4], [1.0]), (3, [5, 6], [0.0, -1.0]),
         (4, [7], [1e-20]), (5, [8], [1.0]), (6, [0], [1.0])]
    A = [(i, np.array(ix), np.array(v)) for i, ix, v in A]
    B = [(i, np.array(ix), np.array(v)) for i, ix, v in B]
    want = sv.multiply_sparse(A, B)
    got = _coo(_mat(A, 3, 7).multiplySparse(_mat(B, 7, 9)))
    _assert_bits(got, want)
    d = {(int(i), int(j)): x for i, j, x in zip(*got)}
    assert d[(0, 0)] == 0.0 and not np.signbit(d[(0, 0)])    # 2 - 2: an exact cancellation stays an entry
    assert np.signbit(d[(0, 4)])                              # the lone product -0.0 * 1.0
    assert np.isnan(d[(0, 5)]) and d[(0, 6)] == -np.inf      # inf * 0 and inf * -1
    assert d[(0, 7)] == f32(1e-20) * f32(1e-20) and d[(0, 7)] != 0   # a float32 subnormal, not flushed
    assert d[(0, 8)] == np.inf                                # 3.5e38 rounds to float overflow
    assert d[(1, 2)] == 0.0 and (2, 0) in d and np.isnan(d[(2, 0)])


def test_empty_sides_and_zero_density():
    import marlin_b200 as mb
    A = [(0, np.array([1]), np.array([2.0])), (2, np.zeros(0, np.int64), np.zeros(0))]
    B = [(0, np.array([0]), np.array([1.0]))]                 # B's row 1 is absent
    cm = _mat(A, 3, 2).multiplySparse(_mat(B, 2, 3))
    assert len(cm.rows) == 0
    z = mb.MTUtils.randomSpaVecMatrix(None, 9, 10, 0.05, seed=3)   # s = 0: empty rows
    assert z.block.nnz == 0 and z.elementsCount() == 9
    assert len(z.multiplySparse(mb.MTUtils.randomSpaVecMatrix(None, 10, 4, 0.5, seed=4)).rows) == 0
    assert np.array_equal(z.toDenseVecMatrix().toBreeze(), np.zeros((9, 10)))


def test_to_dense_vec_matrix_matches_to_breeze():
    rng = np.random.default_rng(8)
    rows = [(i, np.sort(rng.choice(30, 5, replace=False)), rng.standard_normal(5)) for i in (7, 2, 11, 5)]
    m = _mat(rows, 13, 30)
    d = m.toDenseVecMatrix()
    assert sorted(d.ids.tolist()) == list(range(13))
    assert np.array_equal(d.toBreeze(), m.toBreeze())
    assert np.array_equal(m.toBreeze(), sv.to_dense(rows, 13, 30))


@pytest.mark.parametrize("ld_extra", [0, 3, 8])
def test_to_sparse_vec_matrix_round_trip_on_views(ld_extra):
    import torch
    import marlin_b200 as mb
    rng = np.random.default_rng(ld_extra)
    nr, nc = 37, 45
    dense = np.where(rng.random((nr, nc)) < 0.3, rng.standard_normal((nr, nc)), 0.0)
    dense[0, :3] = [-0.0, np.nan, 0.0]
    dense[5] = 0.0
    ld = nc + ld_extra
    host = np.full((nr, ld), 7.0)
    host[:, :nc] = dense
    buf = torch.from_numpy(host.reshape(-1)).cuda()
    ids = np.arange(nr)[::-1].copy()
    dv = mb.DenseVecMatrix(nRows=nr, nCols=nc, ids=ids, data=mb.SubMatrix(buf=buf, rows=nr, cols=nc, ld=ld, is_transpose=True))
    sp = dv.toSparseVecMatrix()
    rp, ci, va = sp.block.to_host()
    want = sv.dense_to_rows(ids, dense)
    assert np.array_equal(sp.ids, ids)
    for r, (i, ix, v) in enumerate(want):
        assert np.array_equal(ci[rp[r]:rp[r + 1]], ix)
        assert np.array_equal(va[rp[r]:rp[r + 1]], v, equal_nan=True)
    back = sp.toDenseVecMatrix().toBreeze()
    expect = np.zeros((nr, nc))
    expect[ids] = np.where(dense == 0.0, 0.0, dense)
    assert np.array_equal(back, expect, equal_nan=True) and not np.signbit(back[nr - 1, 0])


def test_generator_matches_oracle_and_dense_stream():
    import marlin_b200 as mb
    nr, nc, density, seed = 101, 300, 0.05, 42
    sp = mb.MTUtils.randomSpaVecMatrix(None, nr, nc, density, numPartitions=3, seed=seed)
    want = sv.random_spa_vec_matrix(nr, nc, density, 3, seed)
    rp, ci, va = sp.block.to_host()
    s = int(nc * density)
    assert np.array_equal(sp.ids, np.arange(nr)) and np.array_equal(rp, np.arange(nr + 1) * s)
    for r, (i, ix, v) in enumerate(want):
        assert np.array_equal(ci[r * s:(r + 1) * s], ix)
        assert np.array_equal(va[r * s:(r + 1) * s].view(np.uint64), v.view(np.uint64))
    dense = mb.MTUtils.randomDenVecMatrix(None, nr, s, numPartitions=3, seed=seed).toBreeze()
    assert np.array_equal(va.reshape(nr, s), dense)
    bounds = [0, nr // 3, 2 * nr // 3, nr]
    for p in range(3):
        blk = ci.reshape(nr, s)[bounds[p]:bounds[p + 1]]
        assert np.all(blk == blk[0])


def test_errors():
    import marlin_b200 as mb
    from marlin_b200 import _native as nat
    a = _mat(sv.SUITE_ROWS, 4, 4)
    with pytest.raises(mb.MarlinArgumentError) as e:
        a.multiplySparse(_mat(sv.SUITE_ROWS, 5, 4))
    assert e.value.code == nat.MB_ERR_DIM_MISMATCH
    for density in (0.0, -1.0, math.nan, 1.5):
        with pytest.raises(mb.MarlinArgumentError):
            mb.MTUtils.randomSpaVecMatrix(None, 10, 8, density, seed=1)
    with pytest.raises(mb.MarlinArgumentError):
        _mat([(0, [1, 1], [1.0, 2.0])], 2, 4)
    with pytest.raises(mb.MarlinArgumentError):
        _mat([(0, [2, 1], [1.0, 2.0])], 2, 4)
    with pytest.raises(mb.MarlinArgumentError):
        _mat([(1, [1], [1.0]), (1, [2], [2.0])], 2, 4)
    with pytest.raises(mb.MarlinArgumentError):
        _mat([(2 ** 31, [1], [1.0])], 2 ** 32, 4)


def test_chain_into_coordinate_matrix():
    import marlin_b200 as mb
    A = mb.MTUtils.randomSpaVecMatrix(None, 200, 150, 0.1, seed=5)
    B = mb.MTUtils.randomSpaVecMatrix(None, 150, 120, 0.1, seed=6)
    C = A.multiplySparse(B)
    want = sv.multiply_sparse(*[[(i, ix, v) for i, ix, v in sv.random_spa_vec_matrix(*a, 2, sd)]
                                for a, sd in (((200, 150, 0.1), 5), ((150, 120, 0.1), 6))])
    _assert_bits(_coo(C), want)
    d = C.toDenseVecMatrix().toBreeze()
    assert np.array_equal(d[want[0], want[1]], want[2].astype(np.float64))
    U, P = C.ALS(4, 1, 0.1, 2, 2, seed=1)
    assert np.all(np.isfinite(U.data.toBreeze())) and np.all(np.isfinite(P.data.toBreeze()))


def test_two_ranks_bit_identical_to_one(tmp_path):
    sys.path.insert(0, str(ROOT / "tests"))
    import spvec_gpu_worker as w
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    env = dict(os.environ, SPVEC_WORKER_OUT=str(tmp_path / "c"))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), str(ROOT / "tests" / "spvec_gpu_worker.py")]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900, env=env)
    assert out.returncode == 0, out.stdout[-4000:]
    for r in range(2):
        assert f"rank {r} mismatch raised" in out.stdout and f"rank {r} duplicate raised" in out.stdout
    A, B, m, K, n = w.data()
    one = _coo(_mat(A, m, K).multiplySparse(_mat(B, K, n)))
    parts = [np.load(str(tmp_path / f"c.{r}.npz")) for r in range(2)]
    rows = np.concatenate([p["r"] for p in parts])
    cols = np.concatenate([p["c"] for p in parts])
    vals = np.concatenate([p["v"] for p in parts])
    order = np.lexsort((cols, rows))
    assert np.array_equal(rows[order], one[0]) and np.array_equal(cols[order], one[1])
    assert np.array_equal(vals[order].view(np.uint32), one[2].view(np.uint32))
    assert all(int(p["dense_rows"]) >= 0 for p in parts) and sum(int(p["dense_rows"]) for p in parts) == m


def test_strided_columns_and_sparse_wide_rows():
    """Column ids sharing their low bits (multiples of the hash table sizes) in the warp and CTA bins, and window rows whose
    columns lie far apart in 10^8 columns, so almost every window of their range is empty and skipped."""
    from marlin_b200 import _native as nat
    rng = np.random.default_rng(12)
    n = 10 ** 8
    B = []
    for k in range(300):
        if k < 100:
            ix = np.arange(1, 3) * 512 * (k + 1)                      # 2 entries, multiples of 512
        elif k < 200:
            ix = np.arange(1, 41) * 8192 * (k - 99)                   # 40 entries, multiples of 8192
        else:
            ix = np.sort(rng.choice(n, 60, replace=False))            # 60 entries spread over 10^8 columns
        B.append((k, ix, rng.standard_normal(ix.size)))
    A = [(0, np.arange(0, 100), rng.standard_normal(100)),           # u = 200: warp bin
         (1, np.arange(100, 200), rng.standard_normal(100)),         # u = 4000: CTA bin
         (2, np.arange(200, 300), rng.standard_normal(100)),         # u = 6000: window bin, wide range
         (3, np.concatenate([np.arange(100, 200), [250, 251]]), rng.standard_normal(102))]   # u = 4120: window bin
    assert 200 <= nat.MB_SPVEC_WARP_BOUND < 4000 <= nat.MB_SPVEC_CTA_BOUND < 4120
    _assert_bits(_coo(_mat(A, 4, 300).multiplySparse(_mat(B, 300, n))), sv.multiply_sparse(A, B))


def test_to_dense_keeps_negative_zero_and_tuple_rows():
    """A stored -0.0 stays -0.0 in toDenseVecMatrix (the reference's zero-row add gives +0.0; DESIGN 3.11), and a tuple
    of four (id, SparseVector) rows is read as rows, not as arrays."""
    import marlin_b200 as mb
    from marlin_b200.matrix.sparse_matrix import SparseVector
    rows = tuple((i, SparseVector(3, [i % 3], [-0.0 if i == 0 else float(i)])) for i in range(4))
    m = mb.SparseVecMatrix(rows, 4, 3)
    assert sorted(m.ids.tolist()) == [0, 1, 2, 3] and m.elementsCount() == 4
    d = m.toDenseVecMatrix().toBreeze()
    assert d[0, 0] == 0.0 and np.signbit(d[0, 0]) and d[3, 0] == 3.0

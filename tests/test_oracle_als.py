"""The ALS oracle (tests/als_oracle.py) and the coordinate-file loader, on the CPU."""
import numpy as np
import pytest

from marlin_b200 import _native as nat
from marlin_b200.utils import MTUtils
from tests import als_oracle as ao


def _ratings(nu, npr, per_user, seed):
    rng = np.random.default_rng(seed)
    rows, cols = [], []
    for u in range(nu):
        c = rng.choice(npr, per_user, replace=False)
        rows += [u] * per_user
        cols += list(c)
    vals = rng.uniform(0.5, 5.0, len(rows)).astype(np.float32)
    return np.array(rows), np.array(cols), vals


def test_literal_oracle_gives_every_user_one_factor():
    # deviation 2: all users of a block share one XtX and one Xy; with equal rating counts every user gets one factor
    rows, cols, vals = _ratings(12, 9, 4, 0)
    uid, U, _, _ = ao.als(rows, cols, vals, 3, 2, 0.1, nub=1, npb=2, seed=7, literal=True)
    assert np.array_equal(U, np.broadcast_to(U[0], U.shape))
    _, Uc, _, _ = ao.als(rows, cols, vals, 3, 2, 0.1, nub=1, npb=2, seed=7)
    assert not np.allclose(Uc, Uc[0])


def test_literal_implicit_fails_on_missing_yty():
    rows, cols, vals = _ratings(4, 4, 2, 1)
    with pytest.raises(LookupError):
        ao.als(rows, cols, vals, 2, 1, implicit=True, literal=True)


def test_corrected_oracle_matches_dense_masked_als():
    rows, cols, vals = _ratings(30, 20, 6, 2)
    uid, U, pid, P = ao.als(rows, cols, vals, 4, 0, 0.05, nub=3, npb=4, seed=11)
    R = np.zeros((30, 20))
    M = np.zeros((30, 20))
    R[rows, cols] = vals
    M[rows, cols] = 1
    U0 = np.zeros((30, 4))
    P0 = np.zeros((20, 4))
    U0[uid] = U
    P0[pid] = P
    Ud, Pd = ao.dense_masked_als(R, M, U0, P0, 0.05, 3)
    uid, U3, pid, P3 = ao.als(rows, cols, vals, 4, 3, 0.05, nub=3, npb=4, seed=11)
    assert np.allclose(U3, Ud[uid], rtol=1e-9, atol=1e-11)
    assert np.allclose(P3, Pd[pid], rtol=1e-9, atol=1e-11)


def test_link_order_and_duplicates():
    # user 5 rates products 7, 3, 7 (a duplicate), 4 with 3 product blocks: blocks 0 (3), 1 (4, 7), 2 (none)
    rows = np.array([5, 5, 5, 5, 2])
    cols = np.array([7, 3, 7, 4, 4])
    vals = np.array([1, 2, 3, 4, 5], np.float32)
    L = ao.links(rows, cols, vals, 2, 3)
    assert list(L.ids) == [2, 5]                                    # block 0: 2; block 1: 5
    theirs = ao._positions(cols, 3)
    assert list(theirs) == [3, 4, 7]
    p5 = list(L.ids).index(5)
    seg = slice(L.offsets[p5], L.offsets[p5 + 1])
    assert [int(theirs[p]) for p in L.partners[seg]] == [3, 4, 7, 7]
    assert list(L.ratings[seg]) == [2, 4, 1, 3]                     # duplicates in input order
    assert list(L.work) == [p5, list(L.ids).index(2)]               # heaviest first


def test_id_range_rejected():
    with pytest.raises(ValueError):
        ao.links(np.array([2 ** 31]), np.array([0]), np.array([1.0], np.float32), 1, 1)
    with pytest.raises(ValueError):
        ao.links(np.array([0]), np.array([-1]), np.array([1.0], np.float32), 1, 1)


def test_java_random_and_byteswap():
    g = ao.JavaRandom(42)
    assert g.next_int() == -1170105035                              # new java.util.Random(42).nextInt()
    assert ao.JavaRandom(42).next_double() == 0.7275636800328681   # new java.util.Random(42).nextDouble()
    assert ao.JavaRandom(42).next_gaussian() == 1.1419053154730547
    assert ao.byteswap32(0) == 0
    f = ao.random_factor(10, ao.JavaRandom(1))
    assert abs(np.linalg.norm(f) - 1.0) < 1e-15 and (f >= 0).all()


def test_loader(tmp_path):
    p = tmp_path / "r.data"
    p.write_text("1 2 3.5\n1,3,4\n2, 4, 1.00000005960464477550\n3\t5\t2.5\t881250949\n\n")
    m = MTUtils.loadCoordinateMatrix(None, str(p))
    assert list(m.rows) == [1, 1, 2, 3] and list(m.cols) == [2, 3, 4, 5]
    assert m.values.dtype == np.float32
    assert float(m.values[2]) == 1.0000001192092896                # strtof, not float32(float(s)) = 1.0
    assert float(np.float32(float("1.00000005960464477550"))) == 1.0
    assert list(m.values[[0, 1, 3]]) == [3.5, 4.0, 2.5]
    assert m.numRows() == 4 and m.numCols() == 6
    B = m.toBreeze()
    assert B.shape == (4, 6) and B[3, 5] == 2.5


def test_loader_rejects_bad_input(tmp_path):
    with pytest.raises(nat.MarlinArgumentError):
        MTUtils.loadCoordinateMatrix(None, "relative/path")
    p = tmp_path / "bad.data"
    p.write_text("1 2\n")
    with pytest.raises(nat.MarlinArgumentError):
        MTUtils.loadCoordinateMatrix(None, str(p))

"""mb_pagerank_links, the host logic that turns the example's link rows into the in-link rows the step reads (no GPU):
stable source order, weights, target ranges, empty rows and rejected input."""
import ctypes as C

import numpy as np
import pytest

from marlin_b200 import _native as nat
from tests import pagerank_oracle as po


def _links(n, ids, rowptr, targets, values, t0, t1, damping=0.85):
    ids = np.ascontiguousarray(ids, np.int64)
    rowptr = np.ascontiguousarray(rowptr, np.int64)
    targets = np.ascontiguousarray(targets, np.int32)
    values = np.ascontiguousarray(values, np.float64)
    cap = max(int(rowptr[-1]), 1)
    rp, src, w = np.empty(t1 - t0 + 1, np.int32), np.empty(cap, np.int32), np.empty(cap, np.float64)
    nnz = nat.c_i64()
    nat.check(nat.load().mb_pagerank_links(n, len(ids), ids.ctypes.data, rowptr.ctypes.data, targets.ctypes.data,
                                           values.ctypes.data, t0, t1, damping, rp.ctypes.data, src.ctypes.data,
                                           w.ctypes.data, C.byref(nnz)))
    return rp, src[:nnz.value], w[:nnz.value]


@pytest.mark.parametrize("t0,t1", [(0, 300), (0, 150), (150, 300), (17, 18), (40, 40)])
def test_in_links_match_the_oracle(t0, t1):
    n = 300
    src, dst = po.random_graph(n, seed=t0 * 7 + t1)
    ids, rowptr, cols, vals = po.link_rows(src, dst, n)
    shuffle = np.random.default_rng(t1).permutation(len(ids))          # rows in any order: sources come out ascending
    lens = np.diff(rowptr)[shuffle]
    rp_sh = np.concatenate([[0], np.cumsum(lens)])
    cols_sh = np.concatenate([cols[rowptr[r]:rowptr[r + 1]] for r in shuffle])
    vals_sh = np.concatenate([vals[rowptr[r]:rowptr[r + 1]] for r in shuffle])
    rp, s, w = _links(n, ids[shuffle], rp_sh, cols_sh, vals_sh, t0, t1)
    ref = po.InLinks(ids, rowptr, cols, vals, n)
    a, b = ref.start[t0], ref.start[t1]
    assert np.array_equal(rp, ref.start[t0:t1 + 1] - a)
    assert np.array_equal(s, ref.src[a:b])
    assert np.array_equal(w.view(np.int64), ref.w[a:b].view(np.int64))      # fl(value * damping)
    for k in range(t1 - t0):                                                # stable: sources strictly ascending
        assert np.all(np.diff(s[rp[k]:rp[k + 1]]) > 0)


def test_empty_rows_and_no_rows():
    rp, s, w = _links(4, [2], [0, 0], [], [], 0, 4)
    assert rp.tolist() == [0, 0, 0, 0, 0] and len(s) == 0
    rp, s, w = _links(4, [], [0], [], [], 1, 3)
    assert rp.tolist() == [0, 0, 0]
    rp, s, w = _links(3, [2, 0], [0, 2, 3], [0, 1, 1], [0.5, 0.5, 1.0], 0, 3, damping=2.0)
    assert rp.tolist() == [0, 1, 3, 3] and s.tolist() == [2, 0, 2] and w.tolist() == [1.0, 2.0, 1.0]


@pytest.mark.parametrize("args,needle", [
    ((4, [4], [0, 1], [0], [1.0], 0, 4), "source page 4 is outside"),
    ((4, [-1], [0, 1], [0], [1.0], 0, 4), "source page -1 is outside"),
    ((4, [0], [0, 1], [4], [1.0], 0, 4), "target page 4 of source page 0"),
    ((4, [0], [0, 2], [2, 1], [1.0, 1.0], 0, 4), "not strictly increasing"),
    ((4, [0], [0, 2], [1, 1], [1.0, 1.0], 0, 4), "not strictly increasing"),
    ((4, [1, 1], [0, 1, 2], [0, 1], [1.0, 1.0], 0, 4), "source page 1 has two link rows"),
    ((4, [0], [0, 1], [0], [1.0], 3, 5), "target range"),
    ((4, [0], [0, 1], [0], [1.0], 2, 1), "target range"),
    ((4, [0, 1], [0, 2, 1], [0, 1], [1.0, 1.0], 0, 4), "rowptr decreases"),
])
def test_rejected_input(args, needle):
    with pytest.raises(nat.MarlinArgumentError, match=needle):
        _links(*args)

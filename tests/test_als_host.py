"""The ALS host logic of the library (mb_als_links, mb_als_init_factors; no GPU) against the oracle's restatement."""
import numpy as np
import pytest

from marlin_b200 import _native as nat
from marlin_b200.matrix.coordinate_matrix import _Links
from tests import als_oracle as ao


def _data(seed, nnz=400, hi=97):
    rng = np.random.default_rng(seed)
    rows = rng.integers(0, hi, nnz)
    cols = rng.integers(0, 2 * hi, nnz)
    rows[: nnz // 10] = rows[0]                  # one heavy user, with duplicates of its (row, col) pairs
    cols[: nnz // 20] = cols[0]
    return rows, cols, rng.uniform(-5, 5, nnz).astype(np.float32)


@pytest.mark.parametrize("nb,npb", [(1, 1), (3, 10), (10, 3), (7, 1)])
def test_links_match_oracle(nb, npb):
    rows, cols, vals = _data(nb * 31 + npb)
    for ent, partner, a, b in ((rows, cols, nb, npb), (cols, rows, npb, nb)):
        got = _Links(ent, partner, vals, a, b)
        want = ao.links(ent, partner, vals, a, b)
        assert np.array_equal(got.ids, want.ids)
        assert np.array_equal(got.block_offsets, want.block_offsets)
        assert np.array_equal(got.offsets, want.offsets)
        assert np.array_equal(got.partners, want.partners)
        assert np.array_equal(got.ratings.view(np.int32), want.ratings.view(np.int32))
        assert np.array_equal(got.work, want.work)


def test_links_reject_ids_out_of_range():
    for r, c in (([2 ** 31], [0]), ([0], [-1])):
        with pytest.raises(nat.MarlinArgumentError, match="outside"):
            _Links(np.array(r), np.array(c), np.ones(1, np.float32), 1, 1)


@pytest.mark.parametrize("rank", [1, 2, 10, 33, 128])
def test_init_factors_match_oracle(rank):
    rows, cols, vals = _data(rank, nnz=300)
    for side, (ent, partner, a, b) in enumerate(((rows, cols, 4, 5), (cols, rows, 5, 4))):
        got = _Links(ent, partner, vals, a, b).init_factors(-123456789012345, side, rank)
        want = ao.init_factors(ao.links(ent, partner, vals, a, b), -123456789012345, side, rank)
        assert np.array_equal(got, want)

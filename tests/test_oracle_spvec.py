"""The SparseVecMatrix oracle (tests/spvec_oracle.py) against the reference suite and the literal dataflow, the generator
restatement against the existing sampler and dense generator, and the host-side checks of SparseVecMatrix (no GPU)."""
import math

import numpy as np
import pytest

from tests import sparse_oracle as so
from tests import spvec_oracle as sv


def _random_rows(rng, ids, n_cols, per_row, ints=False):
    rows = []
    for i in ids:
        ix = np.sort(rng.choice(n_cols, size=min(per_row, n_cols), replace=False))
        v = rng.integers(-4, 5, ix.size).astype(np.float64) if ints else rng.standard_normal(ix.size)
        rows.append((int(i), ix, v))
    return rows


def test_suite_sparse_matrix_multiply():
    """DistributedMatrixSuite.scala:152-162: the sparse product of sparseData with itself."""
    rows = [(i, np.array(ix), np.array(v)) for i, ix, v in sv.SUITE_ROWS]
    r, c, v = sv.multiply_sparse(rows, rows)
    got = np.zeros((4, 4))
    got[r, c] = v
    assert np.array_equal(got, sv.SUITE_PRODUCT)
    lit = sv.multiply_sparse_literal(rows, rows)
    assert sorted(lit) == sorted(zip(r.tolist(), c.tolist()))


def test_suite_generate_random_sparse_matrix(oracle):
    """DistributedMatrixSuite.scala:147-150: randomSpaVecMatrix(sc, 10, 8, 0.3) has 10 rows."""
    rows = sv.random_spa_vec_matrix(10, 8, 0.3, 2, seed=11)
    assert len(rows) == 10 and sorted(i for i, _, _ in rows) == list(range(10))
    for _, ix, v in rows:
        assert ix.size == 2 and np.all(np.diff(ix) > 0) and ix.max() < 8 and np.all((v >= 0) & (v < 1))


def test_fixed_order_is_the_literal_dataflow_in_k_order():
    rng = np.random.default_rng(3)
    A = _random_rows(rng, range(40), 60, 9)
    B = _random_rows(rng, range(60), 50, 7)
    r, c, v = sv.multiply_sparse(A, B)
    lit = sv.multiply_sparse_literal(A, B)                 # B's rows in id order: products arrive k ascending
    assert len(lit) == len(r)
    for i, j, x in zip(r, c, v):
        assert lit[(int(i), int(j))].view(np.uint32) == x.view(np.uint32)


def test_literal_shuffle_order_agrees_on_exact_data():
    rng = np.random.default_rng(4)
    A = _random_rows(rng, range(30), 40, 8, ints=True)
    B = _random_rows(rng, range(40), 30, 6, ints=True)
    r, c, v = sv.multiply_sparse(A, B)
    for seed in range(3):
        lit = sv.multiply_sparse_literal(A, B, np.random.default_rng(seed))
        assert {k: float(x) for k, x in lit.items()} == {(int(i), int(j)): float(x) for i, j, x in zip(r, c, v)}


def test_structural_entries_and_signed_zero():
    A = [(0, np.array([0, 1]), np.array([1.0, 1.0])), (1, np.array([0]), np.array([-0.0])), (2, np.array([2]), np.array([5.0]))]
    B = [(0, np.array([0, 1]), np.array([0.0, 2.0])), (1, np.array([1]), np.array([-2.0])), (2, np.array([3]), np.array([1.0]))]
    r, c, v = sv.multiply_sparse(A, B)
    got = {(int(i), int(j)): x for i, j, x in zip(r, c, v)}
    assert got[(0, 0)] == 0.0 and got[(0, 1)] == 0.0          # a stored zero and an exact cancellation stay entries
    assert np.signbit(got[(1, 0)]) and np.signbit(got[(1, 1)])  # lone products -0.0 * 0.0 and -0.0 * 2.0 stay -0.0
    assert got[(2, 3)] == 5.0 and len(got) == 5


def test_column_set_is_the_existing_sampler(oracle):
    """Partition p's column set is column 0 of the block sampler run with cols = P rows: positions [s*P, s*P + nColumns)."""
    for seed, P, n, s in [(5, 3, 40, 7), (9, 1, 17, 17), (2, 6, 100, 1), (8, 4, 30, 0)]:
        st = oracle.hash_seed(seed)
        assert np.array_equal(sv.column_set(st, s * P, n, s), so.sample_rows(st, n, P, s)[0])


def test_generator_values_are_the_dense_generator_stream(oracle):
    """Row r of a partition takes the values randomDenVecMatrix gives row r of an nRows x s matrix with the same seed."""
    rows = sv.random_spa_vec_matrix(23, 50, 0.1, 3, seed=77)
    dense = oracle.random_den_vec_matrix(23, 5, 3, seed=77)
    for (i, ix, v), (j, d) in zip(rows, sorted(dense.rows, key=lambda t: t[0])):
        assert i == j and np.array_equal(v, d)
    # one set per partition, shared by all its rows
    for lo, hi in [(0, 7), (7, 15), (15, 23)]:
        sets = {tuple(ix) for i, ix, _ in rows if lo <= i < hi}
        assert len(sets) == 1


def test_dense_to_rows_keeps_nan_and_drops_signed_zeros():
    d = np.array([[0.0, -0.0, np.nan, 2.0], [0.0, 0.0, 0.0, 0.0]])
    (i0, ix0, v0), (i1, ix1, v1) = sv.dense_to_rows([3, 5], d)
    assert list(ix0) == [2, 3] and np.isnan(v0[0]) and v0[1] == 2.0 and ix1.size == 0


@pytest.mark.parametrize("density", [0.0, -0.5, math.nan, 1.2])
def test_column_count_rejects(density):
    import marlin_b200 as mb
    with pytest.raises(mb.MarlinArgumentError):
        mb.matrix.sparse_matrix.column_count(8, 8, density)


def test_column_count_truncates_like_the_jvm():
    from marlin_b200.matrix.sparse_matrix import column_count
    assert column_count(8, 8, 0.3) == 2 and column_count(16384, 16384, 1e-3) == 16 and column_count(10, 10, 0.05) == 0


@pytest.mark.parametrize("args, msg", [
    (((np.array([0, 0]), np.array([0, 1, 2]), np.array([0, 1]), np.ones(2)), 4, 4), "repeated row id 0"),
    (((np.array([-1]), np.array([0, 1]), np.array([0]), np.ones(1)), 4, 4), "outside [0, 2147483647]"),
    (((np.array([2 ** 31]), np.array([0, 1]), np.array([0]), np.ones(1)), 2 ** 32, 4), "outside [0, 2147483647]"),
    (((np.array([4]), np.array([0, 1]), np.array([0]), np.ones(1)), 4, 4), "outside [0, 4)"),
    (((np.array([0]), np.array([0, 2]), np.array([2, 1]), np.ones(2)), 4, 4), "increasing"),
    (((np.array([0]), np.array([0, 2]), np.array([1, 1]), np.ones(2)), 4, 4), "increasing"),
    (((np.array([0]), np.array([0, 1]), np.array([4]), np.ones(1)), 4, 4), "column id"),
])
def test_constructor_rejects(args, msg):
    import marlin_b200 as mb
    with pytest.raises(mb.MarlinArgumentError) as e:
        mb.SparseVecMatrix(*args)
    assert msg in str(e.value)

"""CPU tests of the sparse-block yardstick (tests/sparse_oracle.py) and of the library's pure host logic for sparse
blocks: the four LocalMatrixSuite cases, the defect of the reference's multSparseDense, the generator's properties, and
the column count / structure checks with their messages."""
import numpy as np
import pytest

from marlin_b200 import _native as nat
from marlin_b200.matrix.sparse_matrix import SparseMatrix, SparseVector, check_csc, column_count

from tests import sparse_oracle as so

# LocalMatrixSuite.scala:8-72: the sparse matrix, the dense matrix and the four expected results
SP_COLS = [([1], [1.0]), ([0, 3], [2.0, 1.0]), ([0], [3.0]), ([2], [4.0])]
DENSE = np.array([[0.0, 1.0, 2.0, 3.0], [2.0, 3.0, 4.0, 5.0], [3.0, 2.0, 1.0, 0.0], [1.0, 1.0, 1.0, 1.0]])
EXPECTED_TO_DENSE = np.array([[0.0, 2.0, 3.0, 0.0], [1.0, 0.0, 0.0, 0.0], [0.0, 0.0, 0.0, 4.0], [0.0, 1.0, 0.0, 0.0]])
EXPECTED_DENSE_SPARSE = np.array([[1.0, 3.0, 0.0, 8.0], [3.0, 9.0, 6.0, 16.0], [2.0, 6.0, 9.0, 4.0], [1.0, 3.0, 3.0, 4.0]])
EXPECTED_SPARSE_SPARSE = np.array([[2.0, 0.0, 0.0, 12.0], [0.0, 2.0, 3.0, 0.0], [0.0, 4.0, 0.0, 0.0], [1.0, 0.0, 0.0, 0.0]])
EXPECTED_SPARSE_DENSE = np.array([[13.0, 12.0, 11.0, 10.0], [0.0, 1.0, 2.0, 3.0], [4.0, 4.0, 4.0, 4.0], [2.0, 3.0, 4.0, 5.0]])


def suite_matrix() -> SparseMatrix:
    return SparseMatrix(4, 4, [SparseVector(4, i, v) for i, v in SP_COLS])


def suite_csc():
    return (4, 4, *suite_matrix().to_csc())


def test_local_matrix_suite_cases_exact():
    S = suite_csc()
    assert np.array_equal(so.to_dense(S), EXPECTED_TO_DENSE)
    assert np.array_equal(so.mult_dense_sparse(DENSE, S), EXPECTED_DENSE_SPARSE)
    assert np.array_equal(so.spgemm(S, S), EXPECTED_SPARSE_SPARSE)
    assert np.array_equal(so.mult_sparse_dense(S, DENSE), EXPECTED_SPARSE_DENSE)
    assert np.array_equal(so.mult_sparse_dense_literal(S, DENSE), EXPECTED_SPARSE_DENSE)


def test_restatements_are_the_true_products():
    rng = np.random.default_rng(3)
    A, B = so.random_csc(rng, 37, 41, 0.2, empty_cols=0.2), so.random_csc(rng, 41, 29, 0.3)
    D = rng.standard_normal((23, 37))
    E = rng.standard_normal((41, 19))
    Ad, Bd = so.to_dense(A), so.to_dense(B)
    assert np.allclose(so.mult_dense_sparse(D, A), D @ Ad, rtol=1e-13, atol=1e-13)
    assert np.allclose(so.mult_sparse_dense(A, E), Ad @ E, rtol=1e-13, atol=1e-13)
    assert np.allclose(so.spgemm(A, B), Ad @ Bd, rtol=1e-13, atol=1e-13)


def test_literal_sparse_dense_departs_beyond_32():
    """The reference reads B(bi + k, i) where it means B(bk + k, i) (LibMatrixMult.scala:60): right for K, N <= 32 only."""
    rng = np.random.default_rng(5)
    A = so.random_csc(rng, 8, 32, 0.4)
    B = rng.standard_normal((32, 32))
    assert np.array_equal(so.mult_sparse_dense_literal(A, B), so.mult_sparse_dense(A, B))
    A33 = so.random_csc(rng, 8, 33, 0.4)
    B33 = rng.standard_normal((33, 8))                       # K = 33: the second k-block re-reads rows 0.. of B
    assert not np.array_equal(so.mult_sparse_dense_literal(A33, B33), so.mult_sparse_dense(A33, B33))
    Bn = rng.standard_normal((32, 33))                       # N = 33: column 32 reads past the end of B's data
    with pytest.raises(IndexError):
        so.mult_sparse_dense_literal(A, Bn)
    Bw = rng.standard_normal((16, 40))                       # N = 40, K = 16: columns 32.. read the wrong elements
    A16 = so.random_csc(rng, 8, 16, 0.5)
    try:
        assert not np.array_equal(so.mult_sparse_dense_literal(A16, Bw), so.mult_sparse_dense(A16, Bw))
    except IndexError:
        pass


def test_dense_sparse_copy_case_keeps_negative_zero():
    A = np.array([[-0.0, 2.0], [3.0, -0.0]])
    S = (2, 2, np.array([0, 1, 2], np.int32), np.array([0, 1], np.int32), np.array([1.0, 2.0]))
    out = so.mult_dense_sparse(A, S)
    assert np.signbit(out[0, 0]) and not np.signbit(out[1, 1])          # copy keeps -0.0; 0.0 + 2 * -0.0 is +0.0


def test_generator_properties(oracle):
    rows, cols = 57, 23
    for seed in (1, 42):
        for density in (0.05, 0.4, 1.0, 2.0):
            s = so.column_count(cols, density)
            _, _, cp, ri, va = so.sparse_block(seed, rows, cols, s)
            assert np.array_equal(cp, np.arange(cols + 1) * s)
            for j in range(cols):
                col = ri[cp[j]:cp[j + 1]]
                assert col.size == s and np.all(np.diff(col) > 0) and (s == 0 or (col[0] >= 0 and col[-1] < rows))
            # values: the prefix of the stream the dense generator gives the same block
            assert np.array_equal(va, oracle.uniform_stream(seed, 0, rows * cols)[: s * cols])
    # every row is reachable and the choice is roughly uniform
    _, _, cp, ri, _ = so.sparse_block(7, 40, 400, so.column_count(400, 0.01))
    counts = np.bincount(ri, minlength=40)
    assert counts.min() > 0 and counts.sum() == 400 * 4


def test_generator_blocks_do_not_depend_on_ranks(oracle):
    """Block b is generated from the b-th partition seed alone, so 1, 2 and 3 ranks produce the same blocks."""
    from marlin_b200 import comm
    seeds = oracle.java_random_longs(99, 6)
    whole = {b: so.sparse_block(seeds[b], 30, 20, 3) for b in range(6)}
    for ws in (1, 2, 3):
        got = {}
        for rank in range(ws):
            for b in range(6):
                if comm.elem_owner(b // 3, b % 3, 3, ws) == rank:
                    got[b] = so.sparse_block(seeds[b], 30, 20, 3)
        assert sorted(got) == list(range(6))
        for b in range(6):
            assert all(np.array_equal(x, y) for x, y in zip(got[b][2:], whole[b][2:]))


def test_column_count_truncates_like_the_jvm():
    for cols, d in [(1000, 0.001), (100, 0.07), (3, 0.3333333333333333), (4096, 1e-4), (10, 0.29)]:
        assert column_count(10**6, cols, d) == int(float(cols) * d)
    assert column_count(10, 100, 0.1) == 10
    assert column_count(5, 3, 0.2) == 0                    # (3 * 0.2).toInt == 0: empty columns, as in the reference


@pytest.mark.parametrize("density", [0.0, -0.5, float("nan")])
def test_column_count_rejects_non_positive_density(density):
    with pytest.raises(nat.MarlinArgumentError, match="density of sparse blocks must be positive") as e:
        column_count(10, 10, density)
    assert e.value.code == nat.MB_ERR_INVALID_ARG


def test_column_count_rejects_more_rows_than_the_block_has():
    with pytest.raises(nat.MarlinArgumentError, match="11 non-zeros per column asked of a block with 10 rows"):
        column_count(10, 110, 0.1)


@pytest.mark.parametrize("colptr,rowidx,msg", [
    ([1, 1], [0], "colptr\\[0\\] is 1"),
    ([0, 2, 1], [0], "colptr decreases at column 1"),
    ([0, 2], [1, 1], "not strictly increasing"),
    ([0, 2], [1, 0], "not strictly increasing"),
    ([0, 1], [4], "outside \\[0, 4\\)"),
    ([0, 1], [-1], "outside"),
    ([0, 1], [0, 1], "colptr ends at 1, nnz is 2"),
])
def test_structure_checks(colptr, rowidx, msg):
    cols = len(colptr) - 1
    with pytest.raises(nat.MarlinArgumentError, match=msg):
        check_csc(4, cols, np.array(colptr), np.array(rowidx))


def test_sparse_matrix_to_csc():
    cp, ri, va = suite_matrix().to_csc()
    assert cp.tolist() == [0, 1, 3, 4, 5] and ri.tolist() == [1, 0, 3, 0, 2] and va.tolist() == [1.0, 2.0, 1.0, 3.0, 4.0]
    with pytest.raises(nat.MarlinArgumentError, match="not strictly increasing"):
        SparseMatrix(4, 1, [SparseVector(4, [3, 0], [1.0, 2.0])]).to_csc()     # the reference would accept this unchecked

"""CPU tests: tests/dms_api_oracle.py against the expected matrices of the reference's DistributedMatrixSuite ("slice the
matrix" :207-223, "repeat by row and column" :354-374), and the pure host logic of the norms (mb_norm_mode, mb_norm_fro)
against it."""
import ctypes as C
import math

import numpy as np
import pytest

from marlin_b200 import _native as nat
from tests import dms_api_oracle as do
from tests import marlin_cases as mc

A = mc.EXPECTED_DENSE


def test_slice_the_matrix_suite_case():                    # DMS.scala:207-223
    assert np.array_equal(do.slice_by_row(A, 1, 2), np.array([[2.0, 3.0, 4.0, 5.0], [3.0, 2.0, 1.0, 0.0]]))
    assert np.array_equal(do.slice_by_column(A, 1, 2), np.array([[1.0, 2.0], [3.0, 4.0], [2.0, 1.0], [1.0, 1.0]]))
    assert np.array_equal(do.get_sub_matrix(A, 1, 2, 1, 2), np.array([[3.0, 4.0], [2.0, 1.0]]))


def test_repeat_suite_case():                              # DMS.scala:354-374
    expected1 = np.array([[0.0, 1.0, 2.0, 3.0, 0.0, 1.0, 2.0, 3.0], [2.0, 3.0, 4.0, 5.0, 2.0, 3.0, 4.0, 5.0],
                          [3.0, 2.0, 1.0, 0.0, 3.0, 2.0, 1.0, 0.0], [1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0]])
    expected2 = np.vstack([A, A])
    assert np.array_equal(do.repeat_by_row(A, 2), expected1)
    assert np.array_equal(do.repeat_by_column(A, 2), expected2)
    with pytest.raises(do.Require, match=r"^repeat times: 0 illegal$"):
        do.repeat_by_row(A, 0)


def test_require_messages():
    for call, msg in [(lambda: do.slice_by_row(A, 1, 4), "start row or end row mismatch the matrix num of rows"),
                      (lambda: do.slice_by_row(A, 2, 1), "start row or end row mismatch the matrix num of rows"),
                      (lambda: do.slice_by_column(A, 0, 4), "start column or end column mismatch the matrix num of columns"),
                      (lambda: do.get_sub_matrix(A, 0, 4, 0, 1), "start row or end row dismatch the matrix num of rows"),
                      (lambda: do.get_sub_matrix(A, 0, 1, 2, 1), "start column or end column dismatch the matrix num of columns")]:
        with pytest.raises(do.Require) as e:
            call()
        assert str(e.value) == msg


def test_norms_of_the_suite_matrix():
    assert do.norm(A, "1") == 9.0                          # column sums 6, 7, 8, 9
    assert do.norm(A, "inf") == 14.0                       # row sums 6, 14, 6, 4
    assert do.norm(-A, "inf") == 14.0                      # of |a|: the reference would give -4.0
    assert do.norm(A, "fro") == math.sqrt(float((A * A).sum()))


def test_cbind_and_element_multiply():
    rows_a = {0: [1.0, 2.0], 1: [3.0, 4.0], 2: [5.0, 6.0]}
    rows_b = {0: [7.0], 2: [8.0]}
    got = do.cbind_rows(rows_a, rows_b)
    assert sorted(got) == [0, 2] and list(got[2]) == [5.0, 6.0, 8.0]
    prod = do.element_multiply({(0, 0): [[2.0]], (0, 1): [[3.0]]}, {(0, 0): [[4.0]], (1, 1): [[5.0]]})
    assert list(prod) == [(0, 0)] and prod[(0, 0)][0, 0] == 8.0


def test_grid_rule():
    assert do.relabel_keeps_grid([2, 2, 2, 2])
    assert not do.relabel_keeps_grid([3, 2, 2, 2])          # cBind of widths 3+2 and 2+2: the grid of 9 is 3,3,3,0
    assert not do.relabel_keeps_grid([3, 2, 3, 2])          # repeatByRow of 3+2: the grid of 10 in 4 is 3,3,3,1
    assert do.relabel_keeps_grid([3, 3, 3, 3]) and do.relabel_keeps_grid([3, 3, 2])


@pytest.mark.parametrize("mode", ["1", "inf", "fro", "2", "Inf", "", "one"])
def test_norm_mode_matches_oracle(mode):
    lib = nat.load()
    kind = C.c_int32(-1)
    rc = lib.mb_norm_mode(mode.encode(), C.byref(kind))
    try:
        want = do.norm_mode(mode)
    except do.Require as e:
        assert rc == nat.MB_ERR_INVALID_ARG
        assert lib.mb_last_error().decode() == str(e) == f"Do not support mode {mode}."
        return
    assert rc == nat.MB_OK and kind.value == want


def test_norm_fro_finish():
    lib = nat.load()

    def fro(*triples):
        acc = np.ascontiguousarray(np.array(triples, dtype=np.float64).reshape(-1))
        out = C.c_double()
        assert lib.mb_norm_fro(acc.ctypes.data_as(nat.c_dp), len(triples), C.byref(out)) == nat.MB_OK
        return out.value

    assert fro((0.0, 25.0, 0.0)) == 5.0
    assert fro((0.0, 9.0, 0.0), (0.0, 16.0, 0.0)) == 5.0                              # rank order: 9 + 16
    sbig, ssml = 2.0 ** -538, 2.0 ** 537
    assert fro((0.0, 0.0, (3e300 * sbig) ** 2 + (4e300 * sbig) ** 2)) == pytest.approx(5e300, rel=1e-15)
    assert fro(((3e-300 * ssml) ** 2 + (4e-300 * ssml) ** 2, 0.0, 0.0)) == pytest.approx(5e-300, rel=1e-15)
    assert fro(((1e-300 * ssml) ** 2, 1.0, 0.0)) == 1.0
    assert math.isnan(fro((0.0, math.nan, 1.0)))
    assert math.isinf(fro((0.0, 1.0, math.inf)))
    assert fro((0.0, 0.0, 0.0)) == 0.0
    assert lib.mb_norm_fro(None, 1, None) == nat.MB_ERR_INVALID_ARG

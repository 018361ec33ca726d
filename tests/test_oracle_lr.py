"""The lr oracle (tests/lr_oracle.py) against a plain numpy loop, and MTUtils.loadSVMDenVecMatrix's parsing against the
oracle's restatement of utils/MTUtils.scala:253-276 (no GPU needed)."""
import math

import numpy as np
import pytest

from tests import lr_oracle as lo


def _numpy_lr(A, step, iters, data_size):
    X = A.copy()
    label = X[:, 0].copy()
    X[:, 0] = 1.0
    w = np.zeros(A.shape[1])
    for i in range(1, iters + 1):
        g = 1.0 / (1.0 + np.exp(-(X @ w))) - label
        w = w - (X * g[:, None]).sum(axis=0) * (step / data_size / math.sqrt(i))
    return w


@pytest.mark.parametrize("m,n,iters", [(1, 1, 3), (5, 2, 1), (40, 7, 10), (200, 33, 25)])
def test_oracle_lr_matches_numpy_loop(m, n, iters):
    rng = np.random.default_rng(m + n)
    A = rng.standard_normal((m, n))
    A[:, 0] = rng.integers(0, 2, m)
    rows = [(i, A[i]) for i in range(m)]
    got = lo.lr(rows, 0.7, iters)
    want = _numpy_lr(A, 0.7, iters, m)
    assert np.abs(got - want).max() <= 1e-12 * max(1.0, np.abs(want).max())


def test_oracle_lr_quirks():
    A = np.array([[1.0, 2.0, -1.0], [0.0, 0.5, 4.0]])
    rows = [(7, A[0]), (2, A[1])]
    assert np.array_equal(lo.lr(rows, 1.0, 0), np.zeros(3))                # iters <= 0: zeros
    w = lo.lr(rows, 1.0, 1)
    # w = 0: gradientMul = 0.5 - label; dataSize = max id + 1 = 8
    delta = np.array([1.0, 2.0, -1.0]) * -0.5 + np.array([1.0, 0.5, 4.0]) * 0.5
    assert np.array_equal(w, -delta * (1.0 / 8 / 1.0))
    assert lo.gradient_mul(1000.0, 0.25) == 0.75 and lo.gradient_mul(-1000.0, 0.25) == -0.25
    with pytest.raises(RuntimeError):
        lo.lr([], 1.0, 1)


def _write(tmp_path, text):
    p = tmp_path / "svm.txt"
    p.write_text(text)
    return p


def test_load_svm_matches_oracle(tmp_path):
    from marlin_b200.utils.mt_utils import MTUtils
    text = "5 1:0.5 3:-2\n0 2:1e3\n\n9\n2 4:7 1:1 4:8\n"
    p = _write(tmp_path, text)
    want = lo.load_svm_lines([l for l in text.split("\n") if l.strip()], 4)
    assert [i for i, _ in want] == [5, 0, 9, 2]
    assert np.array_equal(want[2][1], np.zeros(4))                        # a line with no features: zeros
    assert np.array_equal(want[3][1], [1.0, 0.0, 0.0, 8.0])               # a later entry for an index wins
    try:
        import torch
        gpu = torch.cuda.is_available()
    except Exception:
        gpu = False
    if not gpu:
        return                                                            # the matrix itself lives on the device
    mat = MTUtils.loadSVMDenVecMatrix(None, str(p), 4)
    assert mat.numRows() == 10 and mat.numCols() == 4                     # max index + 1
    dense = mat.toBreeze()
    for i, v in want:
        assert np.array_equal(dense[i], v)


def test_load_svm_rejects_relative_path_and_bad_index(tmp_path):
    from marlin_b200 import _native as nat
    from marlin_b200.utils.mt_utils import MTUtils
    with pytest.raises(nat.MarlinArgumentError, match="the path is not in local file System, HDFS or Tachyon"):
        MTUtils.loadSVMDenVecMatrix(None, "relative/svm.txt", 4)
    p = _write(tmp_path, "0 5:1.0\n")
    with pytest.raises(nat.MarlinArgumentError):
        MTUtils.loadSVMDenVecMatrix(None, str(p), 4)
    p = _write(tmp_path, "0 0:1.0\n")
    with pytest.raises(nat.MarlinArgumentError):
        MTUtils.loadSVMDenVecMatrix(None, str(p), 4)
    with pytest.raises(IndexError):
        lo.load_svm_lines(["0 5:1.0"], 4)

"""CPU restatement of DenseVecMatrix.lr (matrix/DenseVecMatrix.scala:1005-1035) and MTUtils.loadSVMDenVecMatrix
(utils/MTUtils.scala:253-276), step by step: the margin is Breeze `features.dot(weights)` as F2J's ddot computes it
(oracle mo_ddot_f2j), exp is the C library's, the gradients are reduced in row order (one partition) and the update is the
reference's expression.  The test suite's yardstick for the device path; nothing under marlin_b200/ imports it."""
from __future__ import annotations

import math
from typing import Iterable, List, Tuple

import numpy as np

from oracle import reference_model as rm


def _exp(x: float) -> float:
    """java.lang.Math.exp: overflows to Infinity instead of raising."""
    try:
        return math.exp(x)
    except OverflowError:
        return math.inf


def gradient_mul(dot: float, label: float) -> float:
    margin = -1.0 * dot
    return (1.0 / (1.0 + _exp(margin))) - label


def lr(rows: List[Tuple[int, np.ndarray]], step: float, iters: int, n_cols: int = 0, n_rows: int = 0) -> np.ndarray:
    """:1005-1035 over one partition holding `rows` in order."""
    mat = rm.DenseVecMatrix(rows, n_rows, n_cols)
    feature_size = mat.num_cols()
    weights = np.zeros(feature_size)
    data_size = mat.num_rows()
    data = []
    for _, v in mat.rows:
        arr = np.array(v, dtype=np.float64)
        label = arr[0]
        arr[0] = 1.0
        data.append((label, arr))
    for i in range(1, iters + 1):
        delta = None
        for label, features in data:
            g = gradient_mul(rm.vector_dot(features, weights), label)
            gradient = features * g
            delta = gradient if delta is None else delta + gradient
        weights = weights - delta * (step / data_size / math.sqrt(i))
    return weights


def gradient(rows: List[Tuple[int, np.ndarray]], weights: np.ndarray) -> np.ndarray:
    """The body of one iteration over one partition: sum of features * gradientMul in row order."""
    delta = np.zeros(len(weights))
    first = True
    for _, v in rows:
        arr = np.array(v, dtype=np.float64)
        label = arr[0]
        arr[0] = 1.0
        gradient = arr * gradient_mul(rm.vector_dot(arr, weights), label)
        delta = gradient if first else delta + gradient
        first = False
    return delta


def load_svm_lines(lines: Iterable[str], vector_len: int) -> List[Tuple[int, np.ndarray]]:
    """:253-276 on the lines of the input: `line.split(" ")`, head = row index, `i:v` entries 1-based."""
    rows = []
    for line in lines:
        items = line.split(" ")
        while items and items[-1] == "":
            items.pop()
        array = np.zeros(vector_len)
        for item in items[1:]:
            ind, value = item.split(":")[:2]
            i = int(ind) - 1
            if not 0 <= i < vector_len:
                raise IndexError(f"index {i} out of bounds for length {vector_len}")
            array[i] = float(value)
        rows.append((int(items[0]), array))
    return rows

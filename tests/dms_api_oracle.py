"""NumPy restatement of the DistributedMatrix API methods that complete the interface (matrix/DenseVecMatrix.scala:238-252,
928-999; matrix/BlockMatrix.scala:673-705; utils/MTUtils.scala:103-125, 446-491).  A matrix is a dense ndarray, a row set
a dict {row id: row}, a block set a dict {(row, col): block}.  Where the port corrects the reference (DESIGN §3.14) the
function says so and restates the corrected behaviour."""
import math

import numpy as np

NORM_ONE, NORM_INF, NORM_FRO = 0, 1, 2


class Require(ValueError):
    """A `require` (IllegalArgumentException) with the reference's message."""


def norm_mode(mode: str) -> int:
    """:975-999 matches "1" and "inf"; "fro" is the port's (a TODO there); "2" and anything else are rejected."""
    kinds = {"1": NORM_ONE, "inf": NORM_INF, "fro": NORM_FRO}
    if mode not in kinds:
        raise Require(f"Do not support mode {mode}.")
    return kinds[mode]


def _max(values) -> float:
    """RDD.max() with java.lang.Double.compare: a NaN is larger than everything."""
    values = np.asarray(values, dtype=np.float64)
    return math.nan if np.isnan(values).any() else float(values.max())


def norm(a: np.ndarray, mode: str) -> float:
    """Corrected: "1" is the largest column sum of |a| (the reference returns the max of accumulators it never fills),
    "inf" the largest row sum of |a| (the reference sums signed values), "fro" sqrt(sum a^2) without overflow."""
    kind = norm_mode(mode)
    a = np.asarray(a, dtype=np.float64)
    if a.shape[0] == 0:
        raise RuntimeError("empty collection")
    if kind == NORM_ONE:
        return _max(np.abs(a).sum(axis=0))
    if kind == NORM_INF:
        return _max(np.cumsum(np.abs(a), axis=1)[:, -1]) if a.shape[1] else 0.0   # a left fold per row
    s = np.abs(a).max() if a.size else 0.0
    if not np.isfinite(s):
        return math.nan if np.isnan(a).any() else math.inf
    if s == 0.0:
        return 0.0
    return float(s * math.sqrt(float(np.sum((a / s) ** 2))))


def slice_by_row(a: np.ndarray, start: int, end: int) -> np.ndarray:
    """:928-933 with inclusive bounds; end == numRows() (a phantom zero row there) is rejected with the same message."""
    if not (start >= 0 and end < a.shape[0] and start <= end):
        raise Require("start row or end row mismatch the matrix num of rows")
    return a[start:end + 1, :]


def slice_by_column(a: np.ndarray, start: int, end: int) -> np.ndarray:
    """:941-946; end == numCols() (short rows there) is rejected with the same message."""
    if not (start >= 0 and end < a.shape[1] and start <= end):
        raise Require("start column or end column mismatch the matrix num of columns")
    return a[:, start:end + 1]


def get_sub_matrix(a: np.ndarray, r0: int, r1: int, c0: int, c1: int) -> np.ndarray:
    """:956-964; also rejects end == numRows()/numCols() and start > end, with the reference's messages."""
    if not (r0 >= 0 and r1 < a.shape[0] and r0 <= r1):
        raise Require("start row or end row dismatch the matrix num of rows")
    if not (c0 >= 0 and c1 < a.shape[1] and c0 <= c1):
        raise Require("start column or end column dismatch the matrix num of columns")
    return a[r0:r1 + 1, c0:c1 + 1]


def cbind_rows(rows_a: dict, rows_b: dict) -> dict:
    """:238-252 — rows.join(that.rows): an inner join on the row id, each row this ++ that."""
    return {i: np.concatenate([np.asarray(v), np.asarray(rows_b[i])]) for i, v in rows_a.items() if i in rows_b}


def repeat_by_row(a: np.ndarray, times: int) -> np.ndarray:
    """:446-464 — despite the name, every row becomes `times` copies of itself (the reference's BlockMatrix branch keeps
    numCols(); corrected to numCols() * times)."""
    if times <= 0:
        raise Require(f"repeat times: {times} illegal")
    return np.tile(a, (1, times))


def repeat_by_column(a: np.ndarray, times: int) -> np.ndarray:
    """:471-491 — the matrix stacked `times` times: row id + i * numRows()."""
    if times <= 0:
        raise Require(f"repeat times: {times} illegal")
    return np.tile(a, (times, 1))


def element_multiply(blocks_a: dict, blocks_b: dict) -> dict:
    """BlockMatrix.scala:673-680 — blocks.join(other.blocks): matching BlockIDs only.  The reference writes the products
    over this matrix's blocks (`:*=`); the port returns new blocks."""
    return {k: np.asarray(v) * np.asarray(blocks_b[k]) for k, v in blocks_a.items() if k in blocks_b}


def constant(n_rows: int, n_cols: int, value: float) -> np.ndarray:
    """MTUtils.scala:103-125 — zerosDenVecMatrix / onesDenVecMatrix."""
    return np.full((n_rows, n_cols), float(value))


def extents(total: int, parts: int):
    """Block heights (widths) of the ceil-sized grid every BlockMatrix method assumes."""
    step = -(-total // parts)
    return [min(step, total - i * step) for i in range(parts)]


def relabel_keeps_grid(ext) -> bool:
    """Whether block widths (heights) ext, relabelled side by side, are exactly the ceil-sized grid of their sum; where
    they are not the port takes the DenseVecMatrix route instead (DESIGN §3.14)."""
    return all(e > 0 for e in ext) and list(ext) == extents(sum(ext), len(ext))

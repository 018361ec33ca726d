"""MTUtils — the drop-in for edu.nju.pasalab.marlin.utils.MTUtils (utils/MTUtils.scala) on the hot path:
input generators, the split chooser, the text loaders and array conversions.

`sc` (the SparkContext argument of the reference signatures) is accepted and ignored: the "cluster" is the
set of ranks of torch.distributed (one process per GPU).
"""
from __future__ import annotations

import ctypes as C
import math
import os
import re
import time
from fractions import Fraction
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from .. import _native as nat
from .. import comm
from ..matrix.block import BlockID
from ..matrix.block_matrix import BlockMatrix
from ..matrix.coordinate_matrix import CoordinateMatrix
from ..matrix.dense_vec_matrix import DenseVecMatrix
from ..matrix.sparse_matrix import SparseBlock, column_count
from ..matrix.sparse_vec_matrix import SparseVecMatrix
from ..matrix.sub_matrix import SubMatrix
from ..runtime import Runtime, world

_SEP = re.compile(r",\s?|\s+")


def _jdouble(v: float) -> str:
    """java.lang.Double.toString: shortest digits that round-trip, plain decimal for 1e-3 <= |v| < 1e7 and computerized
    scientific notation (d.dddE[-]n) outside that range, always at least one digit after the point.  (JDKs before 19
    print a few values with one digit more than the shortest, JDK-4511638; the shortest form is used here.)"""
    v = float(v)
    if v != v:
        return "NaN"
    if v in (float("inf"), float("-inf")):
        return "Infinity" if v > 0 else "-Infinity"
    if v == 0.0:
        return "-0.0" if math.copysign(1.0, v) < 0 else "0.0"
    from decimal import Decimal
    sign, digs, exp = Decimal(repr(abs(v))).as_tuple()
    digits = "".join(str(d) for d in digs).lstrip("0")
    exp += len(digits) - len(digits.rstrip("0"))
    digits = digits.rstrip("0") or "0"
    lead = len(digits) + exp - 1                        # decimal exponent of the leading digit
    neg = "-" if v < 0 else ""
    if 1e-3 <= abs(v) < 1e7:
        if lead >= 0:
            whole = digits[:lead + 1].ljust(lead + 1, "0")
            frac = digits[lead + 1:] or "0"
        else:
            whole, frac = "0", "0" * (-lead - 1) + digits
        return f"{neg}{whole}.{frac}"
    return f"{neg}{digits[0]}.{digits[1:] or '0'}E{lead}"


# java.lang.Float.valueOf's decimal syntax (FloatingDecimal): optional sign, digits with an optional point, an optional
# exponent, an optional f / F / d / D suffix; or NaN / Infinity
_JFLOAT = re.compile(r"[+-]?(NaN|Infinity|((\d+\.?\d*|\.\d+)([eE][+-]?\d+)?)[fFdD]?)")
_F32_MAX_HALF_UP = Fraction(2 ** 128 - 2 ** 103, 1)      # float32 max + half an ulp: from here the value rounds to infinity


def _parse_float32(s: str) -> np.float32:
    """java.lang.Float.parseFloat: the decimal string rounded once, to nearest even, to float32.  Exact rational arithmetic,
    so it depends on no locale; going through a double (float(s), np.float32(s)) rounds twice and can land one float32 ulp
    off ("1.00000005960464477550" gives 1.0 that way, 1.0000001192092896 correctly)."""
    t = s.strip()
    m = _JFLOAT.fullmatch(t)
    if not m:
        raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, f"java.lang.NumberFormatException: For input string: \"{s}\"")
    neg = t.startswith("-")
    if m.group(1) == "NaN":
        return np.float32("nan")
    if m.group(1) == "Infinity":
        return np.float32("-inf" if neg else "inf")
    q = abs(Fraction(m.group(2)))
    if q >= _F32_MAX_HALF_UP:
        v = np.float32("inf")
    else:
        # float32(float(q)) is within one float32 ulp of the correctly rounded value: pick the nearest of it and its two
        # neighbours, ties to the even significand
        c = np.float32(float(q))
        cands = [np.nextafter(c, np.float32(0)), c, np.nextafter(c, np.float32("inf"))]
        v = min((x for x in cands if np.isfinite(x)),
                key=lambda x: (abs(Fraction(float(x)) - q), int(np.array(x).view(np.uint32)) & 1))
    return np.float32(-v) if neg else np.float32(v)


def _check_path(path: str) -> None:
    if not (path.startswith("hdfs://") or path.startswith("tachyon://") or path.startswith("/") or path.startswith("~/")):
        raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, "the path is not in local file System, HDFS or Tachyon")


class UniformGenerator:
    """utils/RandomDataGenerator.scala:53-65 — U[start, end) from XORShiftRandom.nextDouble."""

    def __init__(self, start: float = 0.0, end: float = 1.0):
        self.start, self.end = float(start), float(end)


class StandardNormalGenerator:
    """utils/RandomDataGenerator.scala:70-82 — mean + sqrt(variance) * nextGaussian() over XORShiftRandom, bit-exact
    (mb_fill_normal).  A negative or NaN variance gives NaN values, as math.sqrt does on the JVM."""

    def __init__(self, mean: float = 0.0, variance: float = 1.0):
        self.mean, self.variance = float(mean), float(variance)


class ZerosGenerator:
    """utils/RandomDataGenerator.scala:29-38 — every value 0.0."""


class OnesGenerator:
    """utils/RandomDataGenerator.scala:40-49 — every value 1.0."""


class PoissonGenerator:
    """utils/RandomDataGenerator.scala:89-101 — Colt's Poisson over DRand.  Not generated here: it calls Math.exp and
    Math.log, which the JVM does not specify bit for bit, so there is no value to match; every generator rejects it."""

    def __init__(self, mean: float):
        self.mean = float(mean)


def _check_distribution(dist, what: str, sparse: bool = False) -> None:
    """MB_ERR_UNSUPPORTED naming the generator, before anything is generated (every rank raises together)."""
    if isinstance(dist, (UniformGenerator, StandardNormalGenerator)):
        return
    name = type(dist).__name__
    if isinstance(dist, (ZerosGenerator, OnesGenerator)):
        if not sparse:
            return
        raise nat.MarlinArgumentError(nat.MB_ERR_UNSUPPORTED, f"{what}: {name} is not supported for sparse rows (every "
                                      "stored value would be the same constant)")
    if isinstance(dist, PoissonGenerator):
        raise nat.MarlinArgumentError(nat.MB_ERR_UNSUPPORTED, f"{what}: PoissonGenerator is not supported (Colt's Poisson "
                                      "calls Math.exp / Math.log, which have no bit-exact definition)")
    raise nat.MarlinArgumentError(nat.MB_ERR_UNSUPPORTED, f"{what}: unsupported distribution {name}")


def _svm_vector(items, vectorLen: int) -> np.ndarray:
    """The `i:v` entries of one SVM-format line as a dense vector: entry i sets element i - 1 (a later entry for the same
    index wins); an index outside 1..vectorLen is rejected (ArrayIndexOutOfBoundsException on the JVM)."""
    vec = np.zeros(vectorLen)
    for item in items:
        ind, val = item.split(":")[:2]
        i = int(ind) - 1
        if not 0 <= i < vectorLen:
            raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, f"index {i} out of bounds for length {vectorLen}")
        vec[i] = float(val)
    return vec


class MTUtils:
    # ------------------------------------------------------------------ seeds / RNG plumbing
    @staticmethod
    def hashSeed(seed: int) -> int:
        """utils/MTUtils.scala:18-21"""
        return int(nat.load().mb_hash_seed(seed))

    @staticmethod
    def _partition_seeds(seed: int, num_partitions: int) -> List[int]:
        out = (C.c_int64 * num_partitions)()
        nat.check(nat.load().mb_partition_seeds(seed, num_partitions, out))
        return [int(v) for v in out]

    @staticmethod
    def _fill(blk: SubMatrix, partition_seed: int, first: int, dist, row_major: bool) -> None:
        """generator.setSeed(partition_seed) and blk's values in fill order (rdd/RandomRDD.scala:70-112), the uniform
        stream from value `first` on; the normal stream always starts at its first value, and Zeros and Ones draw
        nothing."""
        rt = Runtime.get(); rt.sync_stream()
        if isinstance(dist, UniformGenerator):
            nat.check(rt.lib.mb_fill_uniform(rt.ctx, blk.handle(), partition_seed, first, dist.start, dist.end, int(row_major)))
        elif isinstance(dist, StandardNormalGenerator):
            nat.check(rt.lib.mb_fill_normal(rt.ctx, blk.handle(), partition_seed, dist.mean, dist.variance, int(row_major), None))
        else:
            nat.check(rt.lib.mb_block_fill(rt.ctx, blk.handle(), 1.0 if isinstance(dist, OnesGenerator) else 0.0))

    @staticmethod
    def _sparse_block(rows: int, cols: int, density: float, partition_seed: int) -> SubMatrix:
        s = column_count(rows, cols, density)
        blk = SparseBlock.empty(rows, cols, s * cols)
        rt = Runtime.get(); rt.sync_stream()
        nat.check(rt.lib.mb_fill_sparse_uniform(rt.ctx, blk.handle(), partition_seed))
        return SubMatrix(sparse=blk)

    # ------------------------------------------------------------------ generators
    @staticmethod
    def randomDenVecMatrix(sc, nRows: int, nColumns: int, numPartitions: int = 0,
                           distribution=None, seed: Optional[int] = None) -> DenseVecMatrix:
        """utils/MTUtils.scala:63-73 -> RandomDenVecRDD (rdd/RandomRDD.scala:161-182).  Partition p holds rows
        [p*N/P, (p+1)*N/P) (:38-41) and is generated on the GPU that owns it (rank p mod G) from the p-th
        nextLong of java.util.Random(seed); values are bit-identical to the reference's XORShift stream for the
        same seed.  The reference's seed is System.nanoTime() and is not exposed (MTUtils.scala:63-73); the extra
        `seed` keyword makes runs reproducible.  `distribution`: UniformGenerator (the default U[0, 1)),
        StandardNormalGenerator, ZerosGenerator or OnesGenerator."""
        dist_ = distribution or UniformGenerator(0.0, 1.0)
        _check_distribution(dist_, "randomDenVecMatrix")
        if seed is None:
            seed = time.time_ns()
        P, shards, ids_arr, data = MTUtils._row_shard(nRows, nColumns, numPartitions)
        seeds = MTUtils._partition_seeds(seed, P)
        off = 0
        for p, s, e in shards:
            view = data.slice(off, off + (e - s), 0, nColumns)
            MTUtils._fill(view, seeds[p], 0, dist_, row_major=True)
            off += e - s
        return DenseVecMatrix(ids=ids_arr, data=data, nRows=nRows, nCols=nColumns)

    @staticmethod
    def _row_shard(nRows: int, nColumns: int, numPartitions: int = 0):
        """The row layout of the dense generators (rdd/RandomRDD.scala:38-41, 161-182): P partitions (numPartitions, or
        the number of ranks, at least 2 on one rank), partition p holds rows [p*N/P, (p+1)*N/P) and lives on rank p mod G.
        Returns (P, [(p, start, end) of this rank], the row ids of this rank, an uninitialised row-major fp64 shard of
        them or None)."""
        rank, ws = world()
        P = numPartitions if numPartitions > 0 else max(ws, 2 if ws == 1 else ws)
        rt = Runtime.get()
        shards, ids = [], []
        start = 0
        for p in range(P):
            end = ((p + 1) * nRows) // P
            if p % ws == rank and end > start:
                shards.append((p, start, end))
                ids.append(np.arange(start, end, dtype=np.int64))
            start = end
        nloc = sum(e - s for _, s, e in shards)
        buf = torch.empty(nloc * nColumns, dtype=torch.float64, device=rt.device)
        data = SubMatrix(buf=buf, rows=nloc, cols=nColumns, ld=max(1, nColumns), is_transpose=True) if nloc else None
        ids_arr = np.concatenate(ids) if ids else np.zeros(0, dtype=np.int64)
        return P, shards, ids_arr, data

    @staticmethod
    def _constant_rows(nRows: int, nColumns: int, value: float) -> DenseVecMatrix:
        _, _, ids, data = MTUtils._row_shard(nRows, nColumns)
        if data is not None:
            rt = Runtime.get()
            rt.sync_stream()
            nat.check(rt.lib.mb_block_fill(rt.ctx, data.handle(), float(value)))
        return DenseVecMatrix(ids=ids, data=data, nRows=nRows, nCols=nColumns)

    @staticmethod
    def zerosDenVecMatrix(sc, nRows: int, nColumns: int) -> DenseVecMatrix:
        """utils/MTUtils.scala:103-109 — every element 0.0, rows laid out as randomDenVecMatrix lays them out."""
        return MTUtils._constant_rows(nRows, nColumns, 0.0)

    @staticmethod
    def onesDenVecMatrix(sc, nRows: int, nColumns: int) -> DenseVecMatrix:
        """utils/MTUtils.scala:119-125 — every element 1.0, rows laid out as randomDenVecMatrix lays them out."""
        return MTUtils._constant_rows(nRows, nColumns, 1.0)

    @staticmethod
    def repeatByRow(matrix, times: int):
        """utils/MTUtils.scala:446-464.  Despite the name, the COLUMNS repeat: every row becomes `times` copies of itself
        side by side (numCols() * times; the reference keeps numCols() for a BlockMatrix, a deviation corrected here).
        times == 1 returns the matrix itself; times <= 0 is rejected."""
        return MTUtils._repeat(matrix, times, columns=True)

    @staticmethod
    def repeatByColumn(matrix, times: int):
        """utils/MTUtils.scala:471-491 — the matrix stacked `times` times: copy i of row id is row id + i * numRows()."""
        return MTUtils._repeat(matrix, times, columns=False)

    @staticmethod
    def _repeat(matrix, times: int, columns: bool):
        times = int(times)
        if times <= 0:
            raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, f"repeat times: {times} illegal")
        if times == 1:
            return matrix
        if isinstance(matrix, DenseVecMatrix):
            return matrix._repeat_columns(times) if columns else matrix._repeat_rows(times)
        if isinstance(matrix, BlockMatrix):
            return matrix._repeat(times, columns)
        raise nat.MarlinArgumentError(nat.MB_ERR_UNSUPPORTED, f"Do not support this type {type(matrix)} for repeat operation")

    @staticmethod
    def randomSpaVecMatrix(sc, nRows: int, nColumns: int, density: float, numPartitions: int = 0,
                           distribution=None, seed: Optional[int] = None) -> SparseVecMatrix:
        """utils/MTUtils.scala:75-85 -> RandomSpaVecRDD (rdd/RandomRDD.scala:47-65, 136-159): the partitions, seeds and rank
        placement of randomDenVecMatrix.  Every row of partition p has the same s = (int)(nColumns * density) sorted columns
        and takes the next s values of the partition's stream, bit-identical to randomDenVecMatrix's values at the same
        stream positions.  The reference draws the column set from an unseeded java.util.Random; here it is drawn by
        selection sampling from the same stream, after the values (mb_fill_spvec_uniform), so it is a function of
        (seed, partition).  density <= 0 and s > nColumns (where the reference never ends) are rejected.
        `distribution`: UniformGenerator or StandardNormalGenerator (mb_fill_spvec_normal: the values are the first s
        values of each row from the partition's normal stream, the column set is drawn right after the positions they
        consumed)."""
        dist_ = distribution or UniformGenerator(0.0, 1.0)
        _check_distribution(dist_, "randomSpaVecMatrix", sparse=True)
        if nRows <= 0 or nColumns <= 0:
            raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, f"randomSpaVecMatrix: {nRows} x {nColumns}")
        s = column_count(nColumns, nColumns, density)
        rank, ws = world()
        P = numPartitions if numPartitions > 0 else max(ws, 2 if ws == 1 else ws)
        if seed is None:
            seed = time.time_ns()
        seeds = MTUtils._partition_seeds(seed, P)
        bounds = [(p * nRows) // P for p in range(P + 1)]
        for r in range(ws):                                 # every rank checks every rank's shard, so all raise together
            if s * sum(bounds[p + 1] - bounds[p] for p in range(r, P, ws)) > 2 ** 31 - 1:
                raise nat.MarlinArgumentError(nat.MB_ERR_UNSUPPORTED, f"randomSpaVecMatrix: a rank's rows would hold more "
                                              f"than 2^31 - 1 non-zeros ({s} per row)")
        rt = Runtime.get()
        rt.sync_stream()
        ids, rps, cis, vas = [], [], [], []
        start, base = 0, 0
        for p in range(P):
            end = ((p + 1) * nRows) // P
            if p % ws == rank and end > start:
                blk = SparseBlock.empty(nColumns, end - start, s * (end - start))
                if isinstance(dist_, UniformGenerator):
                    nat.check(rt.lib.mb_fill_spvec_uniform(rt.ctx, blk.handle(), seeds[p], dist_.start, dist_.end))
                else:
                    nat.check(rt.lib.mb_fill_spvec_normal(rt.ctx, blk.handle(), seeds[p], dist_.mean, dist_.variance))
                ids.append(np.arange(start, end, dtype=np.int64))
                rps.append(blk.colptr[(1 if rps else 0):] + base)
                cis.append(blk.rowidx)
                vas.append(blk.values)
                base += blk.nnz
            start = end
        if not ids:
            block = SparseBlock(nColumns, 0, torch.zeros(1, dtype=torch.int32, device=rt.device),
                                torch.empty(0, dtype=torch.int32, device=rt.device),
                                torch.empty(0, dtype=torch.float64, device=rt.device))
            return SparseVecMatrix._from_block(np.zeros(0, np.int64), block, nRows, nColumns)
        block = SparseBlock(nColumns, sum(len(i) for i in ids), torch.cat(rps), torch.cat(cis), torch.cat(vas))
        return SparseVecMatrix._from_block(np.concatenate(ids), block, nRows, nColumns)

    @staticmethod
    def randomBlockMatrix(sc, nRows: int, nColumns: int, numByRow: int, numByCol: int, sparseInfo=(False, 1.0),
                          distribution=None, seed: Optional[int] = None, dtype: int = nat.MB_F64) -> BlockMatrix:
        """utils/MTUtils.scala:34-50 -> RandomBlockRDD (rdd/RandomRDD.scala:184-223): one partition per block in
        row-major BlockID order, `BDM.create(rows, cols, Array.fill(rows*cols)(nextValue()))` (column-major).

        sparseInfo = (True, density): sparse blocks (SparseMatrix.rand, Matrices.scala:157-173) with
        s = (int)(block cols * density) U[0,1) values in every column.  The reference draws them from unseeded generators,
        so its blocks change on every run; here block b is a function of (seed, b) alone: its values are positions
        [0, s*cols) of the same XORShift stream the dense generator gives that block, and its rows come from selection
        sampling over the next rows*cols positions (mb_fill_sparse_uniform).  density <= 0 and s > block rows are
        rejected; so is a `distribution`, which the reference ignores for sparse blocks.  Dense blocks take
        randomDenVecMatrix's distributions, filled in fp64 and converted to `dtype` afterwards."""
        sparse, density = bool(sparseInfo[0]), float(sparseInfo[1])
        if sparse and distribution is not None:
            raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, "sparse blocks always draw U[0,1) values: the "
                                          "`distribution` argument is not supported with sparseInfo")
        if sparse and dtype != nat.MB_F64:
            raise nat.MarlinArgumentError(nat.MB_ERR_UNSUPPORTED, "sparse blocks are fp64 only")
        dist_ = distribution or UniformGenerator(0.0, 1.0)
        _check_distribution(dist_, "randomBlockMatrix")
        brs = int(math.ceil(float(nRows) / float(numByRow)))
        bcs = int(math.ceil(float(nColumns) / float(numByCol)))
        by_row, by_col = int(math.ceil(nRows / brs)), int(math.ceil(nColumns / bcs))
        if seed is None:
            seed = time.time_ns()
        seeds = MTUtils._partition_seeds(seed, by_row * by_col)
        rank, ws = world()

        def shape(idx: int) -> Tuple[int, int]:
            rows = brs
            if idx >= (by_row - 1) * by_col and brs * by_row > nRows:
                rows = nRows - brs * (by_row - 1)
            cols = bcs
            if (idx + 1) % by_col == 0 and bcs * by_col > nColumns:
                cols = nColumns - bcs * (by_col - 1)
            return rows, cols

        if sparse:
            # every rank checks every block shape (pure host logic) before any generates, so all raise together
            for rows, cols in sorted({shape(idx) for idx in range(by_row * by_col)}):
                column_count(rows, cols, density)
        blocks = []
        for idx in range(by_row * by_col):
            i, j = divmod(idx, by_col)
            if comm.elem_owner(i, j, by_col, ws) != rank:
                continue
            rows, cols = shape(idx)
            if sparse:
                blocks.append((BlockID(i, j), MTUtils._sparse_block(rows, cols, density, seeds[idx])))
                continue
            blk = SubMatrix.empty(rows, cols, nat.MB_F64)
            MTUtils._fill(blk, seeds[idx], 0, dist_, row_major=False)
            if dtype != nat.MB_F64:
                blk = blk.copy(dtype)
            blocks.append((BlockID(i, j), blk.mark_ready()))
        return BlockMatrix(blocks, nRows, nColumns, by_row, by_col, sparse=sparse)

    @staticmethod
    def randomDistVector(sc, length: int, numSplits: int, distribution=None, seed: Optional[int] = None):
        """utils/MTUtils.scala:86-93 -> RandomDistVectorRDD (rdd/RandomRDD.scala:116-134,103-112): one partition per
        piece, piece i = the first splitLength values of the stream seeded with the i-th nextLong of Random(seed);
        the last piece takes the remainder.  `distribution` as in randomDenVecMatrix."""
        from ..matrix.distributed_vector import DistributedVector
        dist_ = distribution or UniformGenerator(0.0, 1.0)
        _check_distribution(dist_, "randomDistVector")
        if seed is None:
            seed = time.time_ns()
        seeds = MTUtils._partition_seeds(seed, numSplits)
        rank, ws = world()
        split_len = int(math.ceil(float(length) / float(numSplits)))
        pieces = []
        for i in range(numSplits):
            if ws > 1 and i % ws != rank:
                continue
            n = length - split_len * i if i == numSplits - 1 else split_len
            blk = SubMatrix.empty(n, 1, nat.MB_F64)
            MTUtils._fill(blk, seeds[i], 0, dist_, row_major=False)
            pieces.append((i, blk))
        return DistributedVector(pieces, length, numSplits)

    @staticmethod
    def onesDistVector(sc, length: int, numSplits: int):
        """utils/MTUtils.scala:128-134 (OnesGenerator pieces)."""
        from ..matrix.distributed_vector import DistributedVector
        rank, ws = world()
        split_len = int(math.ceil(float(length) / float(numSplits)))
        pieces = []
        for i in range(numSplits):
            if ws > 1 and i % ws != rank:
                continue
            n = length - split_len * i if i == numSplits - 1 else split_len
            blk = SubMatrix.zeros(n, 1, nat.MB_F64)
            pieces.append((i, blk.add(1.0)))
        return DistributedVector(pieces)

    # ------------------------------------------------------------------ split chooser
    @staticmethod
    def splitMethod(m: int, k: int, n: int, cores: int) -> Tuple[int, int, int]:
        """utils/MTUtils.scala:150-175"""
        out = (C.c_int32 * 3)()
        nat.check(nat.load().mb_choose_split(m, k, n, cores, out))
        return out[0], out[1], out[2]

    @staticmethod
    def evaluate(mat) -> None:
        """utils/MTUtils.scala:218-220 — force evaluation; here: wait for the GPU."""
        if Runtime.available():
            torch.cuda.synchronize()

    # ------------------------------------------------------------------ conversions
    @staticmethod
    def arrayToMatrix(sc, array: Sequence[Sequence[float]], partitions: int = 2) -> DenseVecMatrix:
        """utils/MTUtils.scala:402-405 — rows are dealt to ranks like sc.parallelize slices."""
        rank, ws = world()
        n = len(array)
        mine = [(i, array[i]) for i in range(n) if ((i * ws) // max(n, 1)) == rank] if ws > 1 else list(enumerate(array))
        return DenseVecMatrix(mine)

    @staticmethod
    def matrixToArray(mat) -> List[List[float]]:
        """utils/MTUtils.scala:416-438"""
        return mat.toBreeze().tolist()

    # ------------------------------------------------------------------ loaders (next-row (f)-3)
    @staticmethod
    def loadMatrixFile(sc, path: str, minPartitions: int = 4) -> DenseVecMatrix:
        """utils/MTUtils.scala:286-300 — `rowIndex:v,v,...`, separators `,\\s?|\\s+`.  Lines are dealt to ranks in
        contiguous chunks (textFile splits)."""
        _check_path(path)
        files = [path] if os.path.isfile(path) else sorted(os.path.join(path, f) for f in os.listdir(path)
                                                           if not f.startswith((".", "_")))
        lines = []
        for f in files:
            with open(f) as fh:
                lines.extend(l.rstrip("\n") for l in fh if l.strip())
        rank, ws = world()
        n = len(lines)
        lo, hi = (rank * n) // ws, ((rank + 1) * n) // ws
        rows = []
        for line in lines[lo:hi]:
            head, body = line.split(":")
            body = body.strip()
            if body.startswith("DenseVector(") and body.endswith(")"):     # what DenseVecMatrix.saveToFileSystem writes
                body = body[len("DenseVector("):-1]
            rows.append((int(head), np.array([float(t) for t in _SEP.split(body) if t != ""], dtype=np.float64)))
        return DenseVecMatrix(rows)

    @staticmethod
    def loadCoordinateMatrix(sc, path: str, minPartitions: int = 4) -> CoordinateMatrix:
        """utils/MTUtils.scala:228-243 — `row col value` or `row col value timestamp` (MovieLens), fields split on
        `,\\s?|\\s+`; the timestamp is ignored.  value.toFloat rounds the decimal string once, straight to float32
        (Float.parseFloat, C strtof), not through a double.  Lines are dealt to ranks in contiguous chunks; blank lines are
        skipped; any other field count is rejected (a MatchError on the JVM)."""
        _check_path(path)
        files = [path] if os.path.isfile(path) else sorted(os.path.join(path, f) for f in os.listdir(path)
                                                           if not f.startswith((".", "_")))
        lines = []
        for f in files:
            with open(f) as fh:
                lines.extend(l.rstrip("\r\n") for l in fh if l.strip())
        rank, ws = world()
        n = len(lines)
        lo, hi = (rank * n) // ws, ((rank + 1) * n) // ws
        rows, cols, vals = [], [], []
        for line in lines[lo:hi]:
            fields = _SEP.split(line)
            while fields and fields[-1] == "":             # java.lang.String.split drops trailing empty strings
                fields.pop()
            if len(fields) not in (3, 4):
                raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, f"scala.MatchError: a line of {len(fields)} fields: {line!r}")
            rows.append(int(fields[0]))
            cols.append(int(fields[1]))
            vals.append(_parse_float32(fields[2]))
        return CoordinateMatrix((np.array(rows, np.int64), np.array(cols, np.int64), np.array(vals, np.float32)))

    @staticmethod
    def loadSVMDenVecMatrix(sc, path: str, vectorLen: int, minPartitions: int = 4) -> DenseVecMatrix:
        """utils/MTUtils.scala:253-276 — `rowIndex i:v i:v ...` split on single spaces: the first token is the row index
        (not a label), each entry sets element i - 1 of a zero vector of vectorLen (a later entry for the same index
        wins).  numRows() is max row index + 1.  Lines are dealt to ranks in contiguous chunks, as loadMatrixFile does;
        blank lines are skipped.  An index outside 1..vectorLen is rejected (ArrayIndexOutOfBoundsException on the JVM)."""
        _check_path(path)
        vectorLen = int(vectorLen)
        files = [path] if os.path.isfile(path) else sorted(os.path.join(path, f) for f in os.listdir(path)
                                                           if not f.startswith((".", "_")))
        lines = []
        for f in files:
            with open(f) as fh:
                lines.extend(l.rstrip("\r\n") for l in fh if l.strip())
        rank, ws = world()
        n = len(lines)
        lo, hi = (rank * n) // ws, ((rank + 1) * n) // ws
        rows = []
        for line in lines[lo:hi]:
            items = line.split(" ")
            while items and items[-1] == "":                 # java.lang.String.split drops trailing empty strings
                items.pop()
            rows.append((int(items[0]), _svm_vector(items[1:], vectorLen)))
        return DenseVecMatrix(rows, 0, vectorLen)

    @staticmethod
    def loadBlockMatrixFile(sc, path: str, minPartitions: int = 4) -> BlockMatrix:
        """utils/MTUtils.scala:324-340 — `row-col-rows-cols:colmajor,...` (the reference requires an hdfs://,
        tachyon:// or file:// prefix here; a plain absolute path is accepted as well)."""
        p = path[len("file://"):] if path.startswith("file://") else path
        files = [p] if os.path.isfile(p) else sorted(os.path.join(p, f) for f in os.listdir(p) if not f.startswith((".", "_")))
        lines = []
        for f in files:
            with open(f) as fh:
                lines.extend(l.strip() for l in fh if l.strip())
        rank, ws = world()
        blocks = []
        for idx, line in enumerate(lines):
            if idx % ws != rank:
                continue
            head, body = line.split(":")
            r, c, nr, nc = (int(t) for t in head.split("-"))
            arr = np.array([float(t) for t in _SEP.split(body) if t != ""], dtype=np.float64).reshape((nr, nc), order="F")
            blocks.append((BlockID(r, c), SubMatrix(arr)))
        placement = None
        if ws > 1:
            import torch.distributed as dist
            keys = [None] * ws
            dist.all_gather_object(keys, [(b.row, b.column) for b, _ in blocks])
            table = {k: r for r, ks in enumerate(keys) for k in ks}
            placement = lambda r, c, t=table: t[(r, c)]
        return BlockMatrix(blocks, placement=placement, sparse=False)

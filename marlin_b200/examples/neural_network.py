"""examples/NeuralNetwork.scala — `neural_network <input> <iterations> <learningRate> <executors> <blocks on each executor>
<selected blocks on each executor> <layer unit num>`: a two-layer sigmoid network on MNIST in libsvm format (`label i:v ...`,
784 features, ten classes) trained by mini-batch SGD over row blocks, writing `hiddenWeight` and `outputWeight` as CSV.

One iteration is mb_nn_step (include/marlin_b200.h): two fp64 DMMA GEMMs with one fused kernel between them.

Deviations from the reference (DESIGN §3.13):
  - genRandomBlocks draws the selected blocks of an executor without replacement from all of its blocks, from a seeded
    generator.  Breeze's `Uniform(0, blk - 1).sample().toInt` never selects an executor's last block and loops forever when
    selected == blocks.
  - The initial weights are N(0, 0.2) from a seeded numpy generator (Breeze's is seeded from the clock); callers can pass
    weights in.
  - The per-block products are summed in ascending block order (treeReduce follows task completion), CUDA's exp is not
    Math.exp and the GEMMs are DMMA, not F2J: weights agree with the reference within rounding, never bit for bit.  At a
    fixed number of ranks a run gives the same bits every time; across rank counts results agree within rounding.
  - A label outside 0..9, a feature index outside 1..vectorLen or an unparsable line raises MarlinArgumentError.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import re
import sys

import numpy as np
import torch

from .. import _native as nat
from .. import comm
from ..matrix.block_matrix import BlockMatrix
from ..matrix.sub_matrix import SubMatrix
from ..matrix.block import BlockID
from ..runtime import Runtime, world
from ..utils.mt_utils import _check_path, _jdouble, _svm_vector

VECTOR_LEN = 28 * 28
CLASSES = 10
WEIGHT_SIGMA = 0.2      # new Gaussian(0, 0.2)

_WS = re.compile(r"\s+")


def _block_rank(row: int, blkNum: int, ws: int) -> int:
    """NeuralNetworkPartitioner puts block row i in partition i; the executors' contiguous runs of blocks go to ranks in
    contiguous runs."""
    return row * ws // blkNum


def loadMNISTImages(sc, input: str, vectorLen: int, blkNum: int):      # noqa: A002
    """NeuralNetwork.scala:32-84 -> (BlockMatrix of blkNum x 1 row blocks, {BlockID(i, 0): int32 labels of block i}).
    Row k of the file (blank lines skipped) goes to block k // ceil(count / blkNum): what splitMethod, toBlockMatrix and
    DistributedIntVector.toDisVector amount to.  A rank parses and holds the blocks _block_rank gives it."""
    vectorLen, blkNum = int(vectorLen), int(blkNum)
    if blkNum < 1 or vectorLen < 1:
        raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, f"NeuralNetwork: {blkNum} blocks of {vectorLen} features")
    _check_path(input)
    files = [input] if os.path.isfile(input) else sorted(os.path.join(input, f) for f in os.listdir(input)
                                                         if not f.startswith((".", "_")))
    lines = []
    for f in files:
        with open(f) as fh:
            lines.extend(l.strip() for l in fh if l.strip())
    count = len(lines)
    if count == 0:
        raise nat.MarlinError(nat.MB_ERR_EMPTY, "empty collection")
    sub = int(math.ceil(count / blkNum))
    nblk = int(math.ceil(count / sub))
    rank, ws = world()
    blocks, labels = [], {}
    for b in range(nblk):
        if _block_rank(b, nblk, ws) != rank:
            continue
        mine = lines[b * sub: min(count, (b + 1) * sub)]
        X = np.empty((len(mine), vectorLen))
        y = np.empty(len(mine), np.int32)
        for k, line in enumerate(mine):
            items = _WS.split(line)
            try:
                y[k] = int(items[0])
                X[k] = _svm_vector(items[1:], vectorLen)
            except ValueError as e:
                if isinstance(e, nat.MarlinArgumentError):
                    raise
                raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, f"NeuralNetwork: cannot parse line {line[:60]!r}") from e
            if not 0 <= y[k] < CLASSES:
                raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG,
                                              f"NeuralNetwork: label {y[k]} of row {b * sub + k} is outside 0..{CLASSES - 1}")
        blocks.append((BlockID(b, 0), SubMatrix(X)))
        labels[BlockID(b, 0)] = y
    placement = lambda row, col: _block_rank(row, nblk, ws)      # noqa: E731
    return BlockMatrix(blocks, count, vectorLen, nblk, 1, placement=placement, sparse=False), labels


def genRandomBlocks(executors: int, blockEachExecutor: int, selectedEachExecutor: int, rng) -> set:
    """:93-105 — selectedEachExecutor distinct blocks of every executor's blockEachExecutor, drawn without replacement."""
    if selectedEachExecutor > blockEachExecutor:
        raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, "requirement failed: the sampled blocks on each executor should "
                                      "be less than the total blocks on each executor")
    out = set()
    for i in range(executors):
        out.update(int(b) + i * blockEachExecutor for b in rng.choice(blockEachExecutor, size=selectedEachExecutor, replace=False))
    return out


def batchSize(selectedEachExecutor: int, blkEachExecutor: int, dataSize: int) -> int:
    """:216 — (selected.toDouble / blkEachExecutor.toDouble * dataSize).toInt"""
    return int(float(selectedEachExecutor) / float(blkEachExecutor) * dataSize)


def _handles(blocks):
    return (nat.c_blk * len(blocks))(*[b.handle().value for b in blocks])


def train(data: BlockMatrix, labels: dict, iterations: int, learningRate: float, executors: int, blkEachExecutor: int,
          selectedEachExecutor: int, layerNum: int, seed: int = 0, hiddenWeight=None, outputWeight=None):
    """The loop of :204-257 -> (hiddenWeight vectorLen x layerNum, outputWeight layerNum x 10) as numpy arrays.

    One rank runs every iteration on its GPU with the weights resident there (mb_nn_step).  With several ranks each rank
    computes the scaled gradient sums of its selected blocks (mb_nn_gradient, zeros if it holds none); they are exchanged
    and added in rank order on every rank, then subtracted, so all ranks hold the same weights bit for bit."""
    vectorLen, dataSize = data.numCols(), data.numRows()
    layerNum = int(layerNum)
    batch = batchSize(selectedEachExecutor, blkEachExecutor, dataSize)
    if batch <= 0 or layerNum < 1:
        raise nat.MarlinArgumentError(nat.MB_ERR_INVALID_ARG, f"NeuralNetwork: batch size {batch}, {layerNum} hidden units")
    rng = np.random.default_rng(seed)
    W1 = rng.normal(0.0, WEIGHT_SIGMA, (vectorLen, layerNum)) if hiddenWeight is None else np.array(hiddenWeight, np.float64)
    W2 = rng.normal(0.0, WEIGHT_SIGMA, (layerNum, CLASSES)) if outputWeight is None else np.array(outputWeight, np.float64)
    if W1.shape != (vectorLen, layerNum) or W2.shape != (layerNum, CLASSES):
        raise nat.MarlinArgumentError(nat.MB_ERR_DIM_MISMATCH, f"NeuralNetwork: weights of {W1.shape} and {W2.shape}, expected "
                                      f"{(vectorLen, layerNum)} and {(layerNum, CLASSES)}")
    rank, ws = world()
    rt = Runtime.get()
    lib, ctx = rt.lib, rt.ctx
    scale = float(learningRate) / batch
    X = {bid.row: blk for bid, blk in data.blocks}
    XT = {row: blk.transpose() for row, blk in X.items()}        # inputData.mapValues(blk => blk.t), once: X never changes
    dev_labels = {}
    try:
        for bid, y in labels.items():
            y = np.ascontiguousarray(y, np.int32)
            p = C.c_void_p()
            nat.check(lib.mb_nn_labels_upload(ctx, y.ctypes.data, len(y), C.byref(p)))
            dev_labels[bid.row] = p
        W1d, W2d = SubMatrix(W1), SubMatrix(W2)
        for _ in range(int(iterations)):
            mine = [b for b in sorted(genRandomBlocks(executors, blkEachExecutor, selectedEachExecutor, rng)) if b in X]
            xs, xts = _handles([X[b] for b in mine]), _handles([XT[b] for b in mine])
            ls = (C.c_void_p * len(mine))(*[dev_labels[b].value for b in mine])
            rt.sync_stream()
            if ws == 1:
                nat.check(lib.mb_nn_step(ctx, xs, xts, ls, len(mine), W1d.handle(), W2d.handle(), scale))
                continue
            g1, g2 = SubMatrix.zeros(vectorLen, layerNum), SubMatrix.zeros(layerNum, CLASSES)
            if mine:
                nat.check(lib.mb_nn_gradient(ctx, xs, xts, ls, len(mine), W1d.handle(), W2d.handle(), scale, g1.handle(),
                                             g2.handle(), None))
            import torch.distributed as dist
            dev = rt.device if dist.get_backend() == "nccl" else torch.device("cpu")
            g = torch.from_numpy(np.concatenate([g1.toBreeze().reshape(-1, order="F"), g2.toBreeze().reshape(-1, order="F")]))
            sends = [(src, dst, ("nn", src)) for src in range(ws) for dst in range(ws) if src != dst]
            got = comm.exchange(sends, {("nn", rank): g.to(dev)}, lambda key: torch.empty(g.numel(), dtype=torch.float64, device=dev), rank)
            parts = [g.numpy() if r == rank else got[("nn", r)].cpu().numpy() for r in range(ws)]
            total = parts[0].copy()
            for p in parts[1:]:
                total = total + p
            W1 = W1d.toBreeze() - total[:W1.size].reshape(W1.shape, order="F")
            W2 = W2d.toBreeze() - total[W1.size:].reshape(W2.shape, order="F")
            W1d, W2d = SubMatrix(W1), SubMatrix(W2)
        W1, W2 = W1d.toBreeze(), W2d.toBreeze()
        rt.synchronize()
    finally:
        for p in dev_labels.values():
            lib.mb_nn_labels_free(ctx, p)
    return W1, W2


def _csvwrite(path: str, M: np.ndarray) -> None:
    """breeze.linalg.csvwrite: one line per row, comma separated."""
    with open(path, "w") as fh:
        for row in M:
            fh.write(",".join(_jdouble(v) for v in row) + "\n")


def main(args):
    from ._common import millis, start, stop
    if len(args) < 7:
        print("usage: NeuralNetwork <input path> <iterations>  <learningRate> <executors> <block on each executor> "
              "<selected blocks on each executor> {<layer unit num> ...}", file=sys.stderr)
        sys.exit(-1)
    mb, rank = start()
    iterations, learningRate = int(args[1]), float(args[2])
    executors, blkEach, selEach, layerNum = int(args[3]), int(args[4]), int(args[5]), int(args[6])
    t0 = millis()
    data, labels = loadMNISTImages(None, args[0], VECTOR_LEN, executors * blkEach)
    if rank == 0:
        print(f"load mnist image used time: {int(millis() - t0)} millis")
    t0 = millis()
    W1, W2 = train(data, labels, iterations, learningRate, executors, blkEach, selEach, layerNum)
    if rank == 0:
        print(f"{iterations} iterations used time: {int(millis() - t0)} millis")
        _csvwrite("hiddenWeight", W1)
        _csvwrite("outputWeight", W2)
    stop()


if __name__ == "__main__":
    main(sys.argv[1:])

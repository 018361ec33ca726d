"""examples/LogisticRegression.scala:11-75 — `logistic_regression <iterations> <stepSize> <instances> <features>`: logistic
regression by full gradient steps written with the matrix-vector operations, on a random instances x features matrix with
all labels 1.  The reference's quirks are kept: theta starts at ones, stepSize is parsed as an Int, the step divides by
stepSize (not multiplies), and the collected pieces are placed at id * splitLen with splitLen = ceil(length / pieces).
DenseVecMatrix.lr is the fused form of one such step (with the reference's other update rule)."""
import math
import sys

import numpy as np

from ._common import millis, start, stop


def _collect(vec, length, f=lambda v: v):
    """vectors.collect() and the `update(id * splitLen + j, f(v(j)))` reassembly into a vector of ones (:54-60, :62-68):
    positions no piece covers keep their 1."""
    pieces = vec._gather([(i, p.toBreeze().reshape(-1)) for i, p in vec.vectors])
    out = np.ones(length)
    split_len = math.ceil(length / len(pieces))
    for i, v in pieces:
        out[i * split_len:i * split_len + v.shape[0]] = f(v)
    return out


def main(args):
    if len(args) < 4:
        print("usage: logistic_regression <iterations> <stepSize> <instances> <features>")
        sys.exit(-1)
    mb, rank = start()
    iterations, step_size, instances, features = int(args[0]), int(args[1]), int(args[2]), int(args[3])
    cores = 1
    splits = 8 * cores
    inp = mb.MTUtils.randomDenVecMatrix(None, instances, features)
    data = inp.toBlockMatrix(splits, 1)                                       # :35-37
    data_transpose = inp.toBlockMatrix(1, 8).transpose()                     # :39
    if rank == 0:
        print(" all the data are generated!")
    labels = mb.MTUtils.onesDistVector(None, instances, splits)             # :42-44
    theta = np.ones(features)                                                # BDV.ones[Double](features)
    t0 = millis()
    for i in range(1, iterations + 1):
        if rank == 0:
            print(f"in iteration {i}")
        q = data.multiply(theta)                                             # :49: data.multiply(theta)
        h = mb.DistributedVector([(pid, mb.SubMatrix((1.0 / (1.0 + np.exp(-p.toBreeze()))).reshape(-1, 1)))
                                  for pid, p in q.vectors], q.length, q.splitNum)   # the sigmoid map of :49-50
        tt = _collect(labels.substract(h), instances)                       # :54-60
        tmp = data_transpose.multiply(tt)                                    # :61
        denom = ((step_size * instances + 2 ** 31) % 2 ** 32 - 2 ** 31) * math.sqrt(i)   # Int * Int wraps, then * Double
        grad = _collect(tmp, features, lambda v: v / denom)                  # :62-68
        theta = theta - grad
    used = millis() - t0
    if rank == 0:
        print(f"theta content: {', '.join(str(v) for v in theta[:10])}{' ...' if features > 10 else ''}")
        print(f"{iterations} iterations used time {used:.0f} millis")
    stop()


if __name__ == "__main__":
    main(sys.argv[1:])

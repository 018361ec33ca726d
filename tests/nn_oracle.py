"""examples/NeuralNetwork.scala restated step by step in plain float64 numpy: the functions of :109-183, one iteration of
:216-248 with the per-block products scaled and then summed in block order, and the loader's re-chunking (:67-80)."""
import math

import numpy as np

CLASSES = 10


def sigmoid(x):
    with np.errstate(over="ignore"):
        return 1.0 / (1.0 + np.exp(-x))


def dSigmoid(x):
    """:109-111"""
    return (1.0 - sigmoid(x)) * sigmoid(x)


def computeOutputError(output, labels):
    """:119-128 — blk(i, vec(i)) -= 1.0 (on a copy: the reference mutates outputLayerOut in place)."""
    out = output.copy()
    out[np.arange(len(labels)), labels] -= 1.0
    return out


def computeDelta(layer_input, error):
    """:152-162"""
    return dSigmoid(layer_input) * error


def backprop(X, labels, W1, W2):
    """One block: (hiddenLayerOut A1, outputDelta D2, hiddenDelta D1), :222-241."""
    Z1 = X @ W1
    A1 = sigmoid(Z1)
    Z2 = A1 @ W2
    A2 = sigmoid(Z2)
    D2 = computeDelta(Z2, computeOutputError(A2, labels))
    D1 = computeDelta(Z1, D2 @ W2.T)
    return A1, D2, D1


def gradient(blocks, labels, W1, W2, scale):
    """computeWeightUpd for both layers (:171-183, :244-248): each block's product times scale, summed in block order."""
    dW1, dW2 = np.zeros_like(W1), np.zeros_like(W2)
    for X, y in zip(blocks, labels):
        A1, D2, D1 = backprop(X, y, W1, W2)
        dW2 = dW2 + (A1.T @ D2) * scale
        dW1 = dW1 + (X.T @ D1) * scale
    return dW1, dW2


def batch_size(selected, blocks_each, data_size):
    """:216"""
    return int(float(selected) / float(blocks_each) * data_size)


def step(blocks, labels, W1, W2, learning_rate, batch):
    dW1, dW2 = gradient(blocks, labels, W1, W2, learning_rate / batch)
    return W1 - dW1, W2 - dW2


def loss(blocks, labels, W1, W2):
    """Half the summed squared output error, the quantity whose gradient the deltas are."""
    total = 0.0
    for X, y in zip(blocks, labels):
        A2 = sigmoid(sigmoid(X @ W1) @ W2)
        total += 0.5 * float((computeOutputError(A2, y) ** 2).sum())
    return total


def rechunk(count, blk_num):
    """Row ranges of the blocks of loadMNISTImages: ceil(count / blkNum) rows each, the last takes the rest."""
    sub = int(math.ceil(count / blk_num))
    return [(lo, min(count, lo + sub)) for lo in range(0, count, sub)]


def parse_libsvm(lines, vector_len):
    """(features, labels) of `label i:v ...` lines, indices from 1 (:52-64, :73-75)."""
    X = np.zeros((len(lines), vector_len))
    y = np.zeros(len(lines), np.int32)
    for k, line in enumerate(lines):
        items = line.split()
        y[k] = int(items[0])
        for item in items[1:]:
            i, v = item.split(":")
            X[k, int(i) - 1] = float(v)
    return X, y

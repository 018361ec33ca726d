"""The NeuralNetwork oracle (tests/nn_oracle.py) against a case worked by hand, and the host side of
marlin_b200.examples.neural_network: the libsvm loader's re-chunking and errors, genRandomBlocks and the batch size."""
import numpy as np
import pytest

from marlin_b200 import _native as nat
from marlin_b200.examples import neural_network as nn
from tests import nn_oracle as no


def test_oracle_matches_a_hand_computed_step():
    """Rows [a, a] against W1 = [[1, 2], [-1, -2]] give Z1 = 0, and W2 = [v; -v] gives Z2 = 0, so every sigmoid is 0.5:
    D2 = +-0.125, E1(r, h) = s_h t_r with s = (1, -1) and t_r = 0.125 (sum(v) - 2 v[y_r]), D1 = 0.25 E1."""
    a = [np.array([1.0, 2.0, 4.0]), np.array([8.0])]
    y = [np.array([0, 3, 3]), np.array([9])]
    blocks = [np.stack([ab, ab], axis=1) for ab in a]
    v = np.arange(1.0, 11.0)
    W1, W2 = np.array([[1.0, 2.0], [-1.0, -2.0]]), np.stack([v, -v])
    scale = 0.25
    dW1, dW2 = no.gradient(blocks, y, W1, W2, scale)
    s = np.array([1.0, -1.0])
    t = [0.125 * (v.sum() - 2.0 * v[yb]) for yb in y]
    want1 = sum(scale * np.outer([(ab * 0.25 * tb).sum()] * 2, s) for ab, tb in zip(a, t))
    counts = np.bincount(np.concatenate(y), minlength=10)
    want2 = np.outer([1.0, 1.0], scale * 0.5 * 0.125 * (4 - 2.0 * counts))
    assert np.array_equal(dW1, want1) and np.array_equal(dW2, want2)
    assert dW1.any() and dW2.any()
    nW1, nW2 = no.step(blocks, y, W1, W2, 1.0, 4)
    assert np.array_equal(nW1, W1 - want1) and np.array_equal(nW2, W2 - want2)


def test_oracle_gradient_is_the_derivative_of_the_loss():
    rng = np.random.default_rng(0)
    X, y = [rng.standard_normal((6, 5))], [rng.integers(0, 10, 6)]
    W1, W2 = rng.normal(0, 0.2, (5, 3)), rng.normal(0, 0.2, (3, 10))
    dW1, dW2 = no.gradient(X, y, W1, W2, 1.0)
    eps = 1e-6
    for W, dW, idx in ((W1, dW1, (2, 1)), (W2, dW2, (1, 7))):
        Wp, Wm = W.copy(), W.copy()
        Wp[idx] += eps
        Wm[idx] -= eps
        args_p = (Wp, W2) if W is W1 else (W1, Wp)
        args_m = (Wm, W2) if W is W1 else (W1, Wm)
        fd = (no.loss(X, y, *args_p) - no.loss(X, y, *args_m)) / (2 * eps)
        assert abs(fd - dW[idx]) <= 1e-8


def _write(tmp_path, lines):
    p = tmp_path / "mnist.libsvm"
    p.write_text("\n".join(lines) + "\n")
    return str(p)


def test_loader_rechunks_rows_and_labels(tmp_path):
    rng = np.random.default_rng(1)
    lines = []
    for k in range(11):
        idx = sorted(rng.choice(np.arange(1, 7), size=rng.integers(0, 5), replace=False))      # trailing features may be missing
        lines.append(" ".join([str(k % 10)] + [f"{i}:{rng.integers(1, 9) / 4}" for i in idx]))
    lines.insert(4, "")                                                                         # blank lines are skipped
    lines.insert(9, "   ")
    data, labels = nn.loadMNISTImages(None, _write(tmp_path, lines), 8, 4)
    X, y = no.parse_libsvm([l for l in lines if l.strip()], 8)
    bounds = no.rechunk(11, 4)
    assert bounds == [(0, 3), (3, 6), (6, 9), (9, 11)]
    assert (data.numRows(), data.numCols(), data.numBlksByRow(), data.numBlksByCol()) == (11, 8, 4, 1)
    for (bid, blk), (lo, hi) in zip(sorted(data.blocks, key=lambda t: t[0].row), bounds):
        assert bid.column == 0 and np.array_equal(blk.toBreeze(), X[lo:hi])
        assert labels[bid].dtype == np.int32 and np.array_equal(labels[bid], y[lo:hi])
    # fewer blocks than asked for when ceil(count / blkNum) rows each cover the rows earlier
    data, labels = nn.loadMNISTImages(None, _write(tmp_path, lines), 8, 8)
    assert data.numBlksByRow() == len(no.rechunk(11, 8)) == 6 and len(labels) == 6


@pytest.mark.parametrize("line", ["3 9:1.0", "3 0:1.0", "10 1:1.0", "-1 1:1.0", "x 1:1.0", "3 1:abc"])
def test_loader_rejects_bad_lines(tmp_path, line):
    with pytest.raises(nat.MarlinArgumentError):
        nn.loadMNISTImages(None, _write(tmp_path, ["1 1:0.5", line]), 8, 1)


def test_gen_random_blocks_draws_distinct_blocks_of_every_executor():
    rng = np.random.default_rng(3)
    seen = set()
    for _ in range(200):
        sel = nn.genRandomBlocks(3, 4, 2, rng)
        assert len(sel) == 6
        for e in range(3):
            assert len([b for b in sel if e * 4 <= b < (e + 1) * 4]) == 2
        seen |= sel
    assert seen == set(range(12))                          # the last block of an executor is drawn too
    assert nn.genRandomBlocks(2, 3, 3, rng) == set(range(6))         # selected == blocks terminates
    assert nn.genRandomBlocks(2, 3, 0, rng) == set()
    with pytest.raises(nat.MarlinArgumentError):
        nn.genRandomBlocks(2, 3, 4, rng)
    a, b = (nn.genRandomBlocks(4, 8, 3, np.random.default_rng(5)) for _ in range(2))
    assert a == b


@pytest.mark.parametrize("sel,each,size,want", [(2, 4, 4096, 2048), (1, 3, 60000, 20000), (1, 3, 10, 3), (3, 3, 7, 7), (1, 7, 6, 0)])
def test_batch_size(sel, each, size, want):
    assert nn.batchSize(sel, each, size) == no.batch_size(sel, each, size) == want

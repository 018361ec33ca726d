"""The PageRank oracle (tests/pagerank_oracle.py): the sparse sequential formulation is bit-identical to the example run
literally on the reference model, which proves the zero-term argument on the CPU; and the example's loader keeps the
reference's values and row presence (no GPU)."""
import numpy as np
import pytest

from marlin_b200 import _native as nat
from marlin_b200.examples import page_rank as pr
from tests import pagerank_oracle as po


def _dense_rows(ids, rowptr, cols, vals, n):
    out = {}
    for r, page in enumerate(ids):
        v = np.zeros(n)
        v[cols[rowptr[r]:rowptr[r + 1]]] = vals[rowptr[r]:rowptr[r + 1]]
        out[int(page)] = v
    return out


@pytest.mark.parametrize("n", [4, 5, 7, 64, 257, 1000])
def test_sparse_formulation_is_the_dense_example_bit_for_bit(n):
    src, dst = po.random_graph(n, seed=n)
    rows = po.link_rows(src, dst, n)
    links = po.InLinks(*rows, n)
    for iterations in (0, 1, 2, 7, 30):
        want = po.dense(_dense_rows(*rows, n), n, iterations)
        got = links.run(iterations)
        assert [len(p) for p in got] == [len(p) for p in want]
        for g, w in zip(got, want):
            assert np.array_equal(g.view(np.int64), w.view(np.int64)), (n, iterations)


def test_heavy_rows_and_missing_blocks_match_the_dense_example():
    """A target with more in-links than the oracle's position-major layout takes (its per-segment accumulate path), and a
    half of the sources without any out-links (so one block of the dense link matrix does not exist)."""
    n = 5000
    src = np.concatenate([np.arange(2500, n), np.arange(2500, n)])
    dst = np.concatenate([np.zeros(2500, np.int64), np.arange(2500, n) % 97])
    rows = po.link_rows(src, dst, n)
    links = po.InLinks(*rows, n, light=100)
    assert len(links.heavy) == 1
    want = po.dense(_dense_rows(*rows, n), n, 3)
    for g, w in zip(links.run(3), want):
        assert np.array_equal(g, w)


def test_link_rows_keep_the_reference_values(tmp_path):
    """Duplicated lines count in links.size but store their target once; self-links are ordinary; pages without
    out-links have no row; extra tokens are ignored; blank lines are skipped."""
    lines = ["1 2", "1 2", "1 3", "2 2", "4 1 extra tokens", "", "   ", "3\t4", "3 1"]
    path = tmp_path / "links.txt"
    path.write_text("\n".join(lines) + "\n")
    m = pr.loadLinksMatrix(None, str(path), 5)
    ids, rp, ci, va = m._host_rows()
    got = _dense_rows(ids, rp, ci, va, 5)
    want = po.literal_rows([l for l in lines if l.strip()], 5)
    assert sorted(got) == sorted(want) == [0, 1, 2, 3]
    for k in want:
        assert np.array_equal(got[k], want[k])
    assert got[0][1] == 1.0 / 3.0 and got[0][2] == 1.0 / 3.0      # "1 2" twice and "1 3": one entry of 1/3 each
    assert m.nRows == m.nCols == 5


@pytest.mark.parametrize("line,needle", [("1 6", "target page 6"), ("0 2", "source page 0"), ("6 1", "source page 6"),
                                         ("1 -1", "target page -1"), ("1 x", "not a number"), ("1", "no target"),
                                         (" 1 2", "not a number"), ("1.0 2", "not a number")])
def test_loader_rejects_bad_lines(tmp_path, line, needle):
    path = tmp_path / "links.txt"
    path.write_text("1 2\n" + line + "\n")
    with pytest.raises(nat.MarlinArgumentError, match=needle) as e:
        pr.loadLinksMatrix(None, str(path), 5)
    assert repr(line) in str(e.value)


def test_small_graph_errors_follow_the_reference_model():
    """n = 2, 3: one block column against two rank pieces fails the reference's require."""
    for n in (2, 3):
        rows = {0: np.full(n, 1.0 / n)}
        with pytest.raises(ValueError, match="not supported matrix or vector"):
            po.dense(rows, n, 1)
        assert len(po.dense(rows, n, 0)) == 2

"""The compiled host mirror's PageRank (include/marlin_b200.hpp, tests/cpp/pagerank_suite.cpp): a hand-checked graph,
ones for no iterations and the errors, and ranks bit-identical to the Python API's.  It builds with -Werror against the C
ABI with plain g++, refuses to run without a GPU, and passes on an H100."""
import numpy as np
import pytest

from tests.harness import build_cpp, no_gpu_check, run_cpp


def test_cpp_pagerank_builds_and_fails_loudly_without_gpu():
    no_gpu_check(build_cpp("pagerank_suite"))


@pytest.mark.gpu
def test_cpp_pagerank_on_gpu(tmp_path):
    import marlin_b200 as mb
    from marlin_b200.examples import page_rank as pr
    from tests import pagerank_oracle as po
    path = tmp_path / "ranks.txt"
    assert "0 failed checks" in run_cpp(build_cpp("pagerank_suite"), path)
    got = np.loadtxt(path, dtype=np.uint64).reshape(-1, 2)
    n = 1000
    i = np.array([k for k in range(n) if k % 5])
    src = np.concatenate([i, i])
    dst = np.concatenate([(7 * i + 3) % n, (i * i + 1) % n])
    ranks = pr.pageRank(mb.SparseVecMatrix(po.link_rows(src, dst, n), n, n), 12)
    want = np.concatenate([v.toBreeze().reshape(-1) for _, v in sorted(ranks.vectors, key=lambda t: t[0])])
    assert np.array_equal(got[:, 0], np.repeat([0, 1], [500, 500]))
    assert np.array_equal(got[:, 1], want.view(np.uint64))

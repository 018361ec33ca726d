"""The compiled host mirror's SparseVecMatrix (include/marlin_b200.hpp, tests/cpp/sparse_vec_suite.cpp): the two
DistributedMatrixSuite cases, the conversions and the errors, and a product bit-identical to the Python API's.  It builds
with -Werror against the C ABI with plain g++, refuses to run without a GPU, and passes on an H100."""
import numpy as np
import pytest

from tests.harness import build_cpp, no_gpu_check, run_cpp


def test_cpp_spvec_builds_and_fails_loudly_without_gpu():
    no_gpu_check(build_cpp("sparse_vec_suite"))


@pytest.mark.gpu
def test_cpp_spvec_on_gpu(tmp_path):
    import marlin_b200 as mb
    coo = tmp_path / "coo.txt"
    assert "0 failed checks" in run_cpp(build_cpp("sparse_vec_suite"), coo)
    got = np.loadtxt(coo, dtype=np.int64).reshape(-1, 3)
    A = mb.MTUtils.randomSpaVecMatrix(None, 300, 200, 0.05, seed=5)
    B = mb.MTUtils.randomSpaVecMatrix(None, 200, 150, 0.05, seed=6)
    C = A.multiplySparse(B)
    order = np.lexsort((C.cols, C.rows))
    g = got[np.lexsort((got[:, 1], got[:, 0]))]
    assert np.array_equal(g[:, 0], C.rows[order]) and np.array_equal(g[:, 1], C.cols[order])
    assert np.array_equal(g[:, 2].astype(np.uint32), C.values[order].view(np.uint32))

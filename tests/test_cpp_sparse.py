"""The compiled host mirror's sparse blocks (include/marlin_b200.hpp; tests/cpp/local_matrix_suite.cpp, the C++ port of
LocalMatrixSuite): builds with -Werror against the C ABI with plain g++, refuses to run without a GPU, and passes on an
H100."""
import pytest

from tests.harness import build_cpp, no_gpu_check, run_cpp


def test_cpp_sparse_builds_and_fails_loudly_without_gpu():
    no_gpu_check(build_cpp("local_matrix_suite"))


@pytest.mark.gpu
def test_cpp_sparse_on_gpu():
    assert "0 failed checks" in run_cpp(build_cpp("local_matrix_suite"))

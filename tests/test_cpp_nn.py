"""The compiled host mirror's NeuralNetwork step (include/marlin_b200.hpp, tests/cpp/nn_suite.cpp): one step of a case
worked by hand, compared exactly, and the errors.  It builds with -Werror against the C ABI with plain g++, refuses to run
without a GPU, and passes on an H100."""
import pytest

from tests.harness import build_cpp, no_gpu_check, run_cpp


def test_cpp_nn_builds_and_fails_loudly_without_gpu():
    no_gpu_check(build_cpp("nn_suite"))


@pytest.mark.gpu
def test_cpp_nn_on_gpu():
    assert "0 failed checks" in run_cpp(build_cpp("nn_suite"))

"""The compiled host mirror's six-argument computeSVD (include/marlin_b200.hpp, tests/cpp/eigs_suite.cpp): builds with
-Werror against the C ABI with plain g++, refuses to run without a GPU, and passes on an H100."""
import pytest

from tests.harness import build_cpp, no_gpu_check, run_cpp


def test_cpp_eigs_builds_and_fails_loudly_without_gpu():
    no_gpu_check(build_cpp("eigs_suite"))


@pytest.mark.gpu
def test_cpp_eigs_on_gpu():
    assert "0 failed checks" in run_cpp(build_cpp("eigs_suite"))

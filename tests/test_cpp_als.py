"""The compiled host mirror's CoordinateMatrix: ALS, toDenseVecMatrix and MTUtils::loadCoordinateMatrix
(include/marlin_b200.hpp, tests/cpp/als_suite.cpp).  It builds with -Werror against the C ABI with plain g++, refuses to run
without a GPU, and passes on an H100."""
import pytest

from tests.harness import build_cpp, no_gpu_check, run_cpp


def test_cpp_als_builds_and_fails_loudly_without_gpu():
    no_gpu_check(build_cpp("als_suite"))


@pytest.mark.gpu
def test_cpp_als_on_gpu():
    assert "0 failed checks" in run_cpp(build_cpp("als_suite"))

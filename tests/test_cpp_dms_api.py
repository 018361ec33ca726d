"""The compiled host mirror's DistributedMatrix API (include/marlin_b200.hpp, tests/cpp/dms_api_suite.cpp): the reference
suite's "slice the matrix" and "repeat by row and column" cases, cBind, elementMultiply, zeros / ones and norm.  It builds
with -Werror against the C ABI with plain g++, refuses to run without a GPU, and passes on an H100."""
import pytest

from tests.harness import build_cpp, no_gpu_check, run_cpp


def test_cpp_dms_api_builds_and_fails_loudly_without_gpu():
    no_gpu_check(build_cpp("dms_api_suite"))


@pytest.mark.gpu
def test_cpp_dms_api_on_gpu():
    assert "0 failed checks" in run_cpp(build_cpp("dms_api_suite"))

"""The compiled host mirror (include/marlin_b200.hpp): the C++ port of the reference's DistributedMatrixSuite builds
against the C ABI with plain g++, refuses to run without a GPU, and passes on an H100."""
import pytest

from tests.harness import build_cpp, no_gpu_check, run_cpp


def test_cpp_suite_builds_and_fails_loudly_without_gpu():
    no_gpu_check(build_cpp("dms_suite"))


@pytest.mark.gpu
def test_cpp_suite_on_gpu():
    assert "0 failed checks" in run_cpp(build_cpp("dms_suite"))


def test_cpp_rank_program_builds_and_fails_loudly_without_gpu():
    """tests/cpp/dist_multiply.cpp (the compiled caller of the multi-GPU multiply) builds with -Werror against the host mirror
    and, like everything else, refuses to run without a GPU."""
    from tests.test_gpu_dist_cabi import build_cpp_rank_program
    no_gpu_check(build_cpp_rank_program(), 0, 1, "nogpu", 1)

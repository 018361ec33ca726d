"""The compiled host mirror's StandardNormalGenerator overloads (include/marlin_b200.hpp, tests/cpp/random_suite.cpp):
builds with -Werror against the C ABI with plain g++, refuses to run without a GPU, and on an H100 matches the suite's
host restatement of the reference generator value for value."""
import pytest

from tests.harness import build_cpp, no_gpu_check, run_cpp


def build_random_suite():
    return build_cpp("random_suite", extra=("-ffp-contract=off",))       # the JVM never fuses a multiply and an add


def test_cpp_random_builds_and_fails_loudly_without_gpu():
    no_gpu_check(build_random_suite())


@pytest.mark.gpu
def test_cpp_random_on_gpu():
    assert "0 failed checks" in run_cpp(build_random_suite())

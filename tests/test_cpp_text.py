"""The compiled host mirror's matrix-file writers (include/marlin_b200.hpp, tests/cpp/text_suite.cpp): builds with
-Werror against the C ABI with plain g++, refuses to run without a GPU, and on an H100 writes the files the oracle's
line restatements give, byte for byte."""
import math

import numpy as np
import pytest

from tests.harness import build_cpp, no_gpu_check, run_cpp


def build_text_suite():
    return build_cpp("text_suite")


def test_cpp_text_builds_and_fails_loudly_without_gpu(tmp_path):
    no_gpu_check(build_text_suite(), tmp_path)


def value(i, j, cols):
    s = [0.0, -0.0, 1.0, -2.5, 0.001, 9.999999999999998e-4, 1e7, 5e-324, 1.7976931348623157e308, math.nan, math.inf,
         -math.inf, 0.1, 123456.789, 1.0 / 3.0]
    return s[(i * cols + j) % 15] * (-1.0 if i % 2 else 1.0)


@pytest.mark.gpu
def test_cpp_text_on_gpu(oracle, tmp_path):
    assert "0 failed checks" in run_cpp(build_text_suite(), tmp_path)
    ids = [0, 3, 1, 1 << 40, 7, 5, 6]
    vals = [np.array([value(i, j, 5) for j in range(5)]) for i in range(7)]
    om = oracle.DenseVecMatrix(list(zip(ids, vals)))
    assert (tmp_path / "rows" / "part-00000").read_text() == "".join(x + "\n" for x in om.save_lines())
    assert (tmp_path / "rows" / "_description").read_text() == om.description()
    od = oracle.DenseVecMatrix(list(enumerate(vals)))
    ob = od.to_block_matrix(2, 2)
    lines = lambda p: (tmp_path / p / "part-00000").read_text().splitlines(keepends=True)
    assert sorted(lines("blocks")) == sorted(x + "\n" for x in ob.save_block_lines())
    assert sorted(lines("blocks_t")) == sorted(x + "\n" for x in ob.transpose().save_block_lines())
    assert sorted(lines("blocks_rows")) == sorted(x + "\n" for x in od.save_lines())

"""The compiled host mirror's SparseVecMatrix (include/marlin_b200.hpp, tests/cpp/sparse_vec_suite.cpp): the two
DistributedMatrixSuite cases, the conversions and the errors, and a product bit-identical to the Python API's.  It builds
with -Werror against the C ABI with plain g++, refuses to run without a GPU, and passes on an H100."""
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
BIN = ROOT / "scripts" / "bin" / "sparse_vec_suite"


def build_suite() -> Path:
    from marlin_b200 import _native as nat
    nat.load()
    BIN.parent.mkdir(parents=True, exist_ok=True)
    cmd = [shutil.which("g++") or "g++", "-std=c++17", "-O1", "-Wall", "-Werror", f"-I{ROOT / 'include'}",
           str(ROOT / "tests" / "cpp" / "sparse_vec_suite.cpp"), f"-L{ROOT / 'marlin_b200' / 'lib'}", "-lmarlin_b200",
           "-Wl,-rpath,$ORIGIN/../../marlin_b200/lib", "-o", str(BIN)]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert out.returncode == 0, out.stdout
    return BIN


def test_cpp_spvec_builds_and_fails_loudly_without_gpu():
    import torch
    exe = build_suite()
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by test_cpp_spvec_on_gpu")
    out = subprocess.run([str(exe)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=120)
    assert out.returncode == 3
    assert "no CPU fallback" in out.stdout


@pytest.mark.gpu
def test_cpp_spvec_on_gpu(tmp_path):
    import marlin_b200 as mb
    exe = build_suite()
    coo = tmp_path / "coo.txt"
    out = subprocess.run([str(exe), str(coo)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert out.returncode == 0, out.stdout[-3000:]
    assert "0 failed checks" in out.stdout
    got = np.loadtxt(coo, dtype=np.int64).reshape(-1, 3)
    A = mb.MTUtils.randomSpaVecMatrix(None, 300, 200, 0.05, seed=5)
    B = mb.MTUtils.randomSpaVecMatrix(None, 200, 150, 0.05, seed=6)
    C = A.multiplySparse(B)
    order = np.lexsort((C.cols, C.rows))
    g = got[np.lexsort((got[:, 1], got[:, 0]))]
    assert np.array_equal(g[:, 0], C.rows[order]) and np.array_equal(g[:, 1], C.cols[order])
    assert np.array_equal(g[:, 2].astype(np.uint32), C.values[order].view(np.uint32))

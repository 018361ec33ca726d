"""The compiled host mirror's StandardNormalGenerator overloads (include/marlin_b200.hpp, tests/cpp/random_suite.cpp):
builds with -Werror against the C ABI with plain g++, refuses to run without a GPU, and on an H100 matches the suite's
host restatement of the reference generator value for value."""
import shutil
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
BIN = ROOT / "scripts" / "bin" / "random_suite"


def build_random_suite() -> Path:
    from marlin_b200 import _native as nat
    nat.load()
    BIN.parent.mkdir(parents=True, exist_ok=True)
    cmd = [shutil.which("g++") or "g++", "-std=c++17", "-O1", "-ffp-contract=off", "-Wall", "-Werror", f"-I{ROOT / 'include'}",
           str(ROOT / "tests" / "cpp" / "random_suite.cpp"), f"-L{ROOT / 'marlin_b200' / 'lib'}", "-lmarlin_b200",
           "-Wl,-rpath,$ORIGIN/../../marlin_b200/lib", "-o", str(BIN)]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert out.returncode == 0, out.stdout
    return BIN


def test_cpp_random_builds_and_fails_loudly_without_gpu():
    import torch
    exe = build_random_suite()
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by test_cpp_random_on_gpu")
    out = subprocess.run([str(exe)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=120)
    assert out.returncode == 3
    assert "no CPU fallback" in out.stdout


@pytest.mark.gpu
def test_cpp_random_on_gpu():
    exe = build_random_suite()
    out = subprocess.run([str(exe)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert out.returncode == 0, out.stdout[-3000:]
    assert "0 failed checks" in out.stdout

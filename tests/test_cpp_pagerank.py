"""The compiled host mirror's PageRank (include/marlin_b200.hpp, tests/cpp/pagerank_suite.cpp): a hand-checked graph,
ones for no iterations and the errors, and ranks bit-identical to the Python API's.  It builds with -Werror against the C
ABI with plain g++, refuses to run without a GPU, and passes on an H100."""
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
BIN = ROOT / "scripts" / "bin" / "pagerank_suite"


def build_suite() -> Path:
    from marlin_b200 import _native as nat
    nat.load()
    BIN.parent.mkdir(parents=True, exist_ok=True)
    cmd = [shutil.which("g++") or "g++", "-std=c++17", "-O1", "-Wall", "-Werror", f"-I{ROOT / 'include'}",
           str(ROOT / "tests" / "cpp" / "pagerank_suite.cpp"), f"-L{ROOT / 'marlin_b200' / 'lib'}", "-lmarlin_b200",
           "-Wl,-rpath,$ORIGIN/../../marlin_b200/lib", "-o", str(BIN)]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert out.returncode == 0, out.stdout
    return BIN


def test_cpp_pagerank_builds_and_fails_loudly_without_gpu():
    import torch
    exe = build_suite()
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by test_cpp_pagerank_on_gpu")
    out = subprocess.run([str(exe)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=120)
    assert out.returncode == 3
    assert "no CPU fallback" in out.stdout


@pytest.mark.gpu
def test_cpp_pagerank_on_gpu(tmp_path):
    import marlin_b200 as mb
    from marlin_b200.examples import page_rank as pr
    from tests import pagerank_oracle as po
    exe = build_suite()
    path = tmp_path / "ranks.txt"
    out = subprocess.run([str(exe), str(path)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert out.returncode == 0, out.stdout[-3000:]
    assert "0 failed checks" in out.stdout
    got = np.loadtxt(path, dtype=np.uint64).reshape(-1, 2)
    n = 1000
    i = np.array([k for k in range(n) if k % 5])
    src = np.concatenate([i, i])
    dst = np.concatenate([(7 * i + 3) % n, (i * i + 1) % n])
    ranks = pr.pageRank(mb.SparseVecMatrix(po.link_rows(src, dst, n), n, n), 12)
    want = np.concatenate([v.toBreeze().reshape(-1) for _, v in sorted(ranks.vectors, key=lambda t: t[0])])
    assert np.array_equal(got[:, 0], np.repeat([0, 1], [500, 500]))
    assert np.array_equal(got[:, 1], want.view(np.uint64))

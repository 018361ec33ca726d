"""The PageRank kernels in the built library (cuobjdump -sass, no GPU needed): every instance of pagerank_step_kernel
multiplies and adds in fp64 with separate DMUL and DADD (no DFMA: the JVM never contracts a * b + c), and no PageRank
kernel touches local memory."""
import collections
import re
import shutil
import subprocess

import pytest

from marlin_b200 import _native as nat


@pytest.fixture(scope="module")
def kernels():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    nat.load()
    out = subprocess.run([exe, "-sass", str(nat._LIB_PATH)], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=600)
    if out.returncode != 0:
        pytest.skip("cuobjdump unavailable: " + out.stderr[:200])
    res = {}
    for chunk in re.split(r"\n\s*Function : ", out.stdout)[1:]:
        mangled = chunk.split("\n", 1)[0].strip()
        if "pagerank_cu" in mangled:
            res[mangled] = collections.Counter(m.group(1).split(".")[0] for m in
                                               re.finditer(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Za-z0-9_.]*)", chunk))
    return res


def test_step_kernels_multiply_and_add_separately(kernels):
    steps = [v for k, v in kernels.items() if "pagerank_step_kernel" in k]
    assert len(steps) == 2, sorted(kernels)                 # the light-row and the heavy-row instance
    for ops in steps:
        assert ops["DFMA"] == 0
        assert ops["DMUL"] >= 1 and ops["DADD"] >= 1


def test_no_local_memory(kernels):
    assert len(kernels) == 3, sorted(kernels)
    for ops in kernels.values():
        assert ops["LDL"] == 0 and ops["STL"] == 0

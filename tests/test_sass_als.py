"""The ALS kernels in the built library (cuobjdump -sass, no GPU needed): the assembly-only instances of als_kernel add and
multiply with separate DADD / DMUL (no DFMA: the JVM never contracts), and no instance touches local memory."""
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
        if "2mb10als_kernelI" in mangled:          # mb::als_kernel<...>
            res[mangled] = collections.Counter(m.group(1).split(".")[0] for m in
                                               re.finditer(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Za-z0-9_.]*)[^;]*;", chunk))
    return res


def test_assembly_instances_never_fuse(kernels):
    # als_kernel<G, EPT, SOLVE = false>: the mangled template argument list ends in Lb0E
    asm = {k: v for k, v in kernels.items() if "Lb0E" in k}
    assert len(asm) == 5, sorted(kernels)              # one per rank bucket
    for ops in asm.values():
        assert ops["DFMA"] == 0
        assert ops["DMUL"] >= 2 and ops["DADD"] >= 2


def test_no_local_memory(kernels):
    assert len(kernels) == 10
    for ops in kernels.values():
        assert ops["LDL"] == 0 and ops["STL"] == 0

"""The SparseVecMatrix kernels in the built library (cuobjdump -sass, no GPU needed): the product kernels multiply and add
in float32 with separate FMUL and FADD (no FFMA: the JVM never contracts a * b + c), and no spvec kernel touches local
memory."""
import collections
import re
import shutil
import subprocess

import pytest

from marlin_b200 import _native as nat

PRODUCT_KERNELS = ("spvec_warp_kernelILb1E", "spvec_cta_kernelILb1E", "spvec_window_kernelILb1E")


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
        if "spvec_cu" in mangled:
            res[mangled] = collections.Counter(m.group(1).split(".")[0] for m in
                                               re.finditer(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Za-z0-9_.]*)", chunk))
    return res


@pytest.mark.parametrize("needle", PRODUCT_KERNELS)
def test_products_multiply_and_add_separately(kernels, needle):
    fam = [v for k, v in kernels.items() if needle in k]
    assert len(fam) == 1, (needle, sorted(kernels))
    ops = fam[0]
    assert ops["FFMA"] == 0
    assert ops["FMUL"] >= 1 and ops["FADD"] >= 1


def test_no_local_memory(kernels):
    assert len(kernels) == 11, sorted(kernels)
    for ops in kernels.values():
        assert ops["LDL"] == 0 and ops["STL"] == 0

"""The SVD kernels in the built library (cuobjdump -sass, no GPU needed): the Gramian runs the DMMA mainloop fed by TMA,
the reduce-and-mirror pass uses 128-bit accesses, and none of the new kernels spills to local memory."""
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
        res[mangled] = collections.Counter(m.group(1) for m in re.finditer(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Za-z0-9_.]*)", chunk))
    return res


def _count(ops, prefix):
    return sum(v for k, v in ops.items() if k.split(".")[0] == prefix)


def _family(kernels, needle):
    fam = {k: v for k, v in kernels.items() if needle in k}
    assert fam, needle
    return fam


def test_gramian_is_dmma_fed_by_tma(kernels):
    fam = _family(kernels, "syrk_f64_dmma_kernel")
    assert len(fam) == 2                                       # row-shard (N,T) and column-major (T,N) operands
    for name, ops in fam.items():
        assert ops.get("DMMA.8x8x4", 0) == 128, name
        assert _count(ops, "UTMALDG") >= 2 and _count(ops, "SYNCS") >= 10, name
        assert _count(ops, "LDL") == 0 and _count(ops, "STL") == 0, name


def test_svd_kernels_do_not_spill(kernels):
    for needle in ("gram_reduce_mirror_kernel", "jacobi_round_kernel", "jacobi_init_kernel", "jacobi_gather_kernel"):
        for name, ops in _family(kernels, needle).items():
            assert _count(ops, "LDL") == 0 and _count(ops, "STL") == 0, name
    fam = _family(kernels, "gram_reduce_mirror_kernel")
    assert len(fam) == 2                                       # 128-bit or scalar reads of the partials
    for name, ops in fam.items():
        assert any(k.startswith("STG.E.128") for k in ops), name
        if "ILb1E" in name:
            assert any(k.startswith("LDG.E.128") for k in ops), name
    for name, ops in _family(kernels, "jacobi_round_kernel").items():
        assert any(k.startswith("LDG.E.128") for k in ops) and any(k.startswith("STG.E.128") for k in ops), name

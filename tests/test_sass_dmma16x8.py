"""The full-rate fp64 kernels in the built library (cuobjdump -sass, no GPU needed): every fp64 GEMM, grouped and Gramian
kernel that production launches issues DMMA.16x8x4 (mma.sync.m16n8k4, twice the fp64 rate of DMMA.8x8x4 on H100), fed by
the same TMA ring and the same 24 conflict-free LDS.128 per k16 slab as the m8n8k4 reference instances, without spills."""
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


@pytest.mark.parametrize("needle, instances", [("gemm_f64_dmma16x8_kernel", 4),           # the four N/T operand forms
                                               ("gemm_f64_dmma16x8_grouped_kernel", 1),   # the blocked multiply
                                               ("syrk_f64_dmma16x8_kernel", 2)])          # Gramian: (N,T) and (T,N)
def test_fp64_kernels_issue_dmma_16x8x4(kernels, needle, instances):
    fam = {k: v for k, v in kernels.items() if needle in k}
    assert len(fam) == instances, sorted(fam)
    for name, ops in fam.items():
        assert ops.get("DMMA.16x8x4", 0) == 64, (name, ops.get("DMMA.16x8x4"))     # one k16 slab of a 64x32 warp tile
        assert _count(ops, "DMMA") == 64, name                                     # ... and no other DMMA shape
        lds = sum(v for k, v in ops.items() if k.startswith("LDS"))
        assert lds == 24 and all(k.startswith("LDS.128") or not k.startswith("LDS") for k in ops), name
        assert _count(ops, "UTMALDG") >= 2 and _count(ops, "SYNCS") >= 10, name    # TMA loads + mbarrier pipeline
        assert _count(ops, "USETMAXREG") == 2, name                                # producer gives registers to consumers
        assert _count(ops, "LDL") == 0 and _count(ops, "STL") == 0, name           # no spills


def test_reference_instances_are_the_same_kernels_at_m8n8k4(kernels):
    """Each full-rate kernel has its m8n8k4 reference instance (mb_set_dmma_reference) under the older name."""
    for old, new in (("gemm_f64_dmma_kernel", "gemm_f64_dmma16x8_kernel"),
                     ("gemm_f64_dmma_grouped_kernel", "gemm_f64_dmma16x8_grouped_kernel"),
                     ("syrk_f64_dmma_kernel", "syrk_f64_dmma16x8_kernel")):
        ref = {k.split(old, 1)[1]: v for k, v in kernels.items() if old in k}
        full = {k.split(new, 1)[1]: v for k, v in kernels.items() if new in k}
        assert ref and set(ref) == set(full), (old, sorted(ref), sorted(full))   # same template instances
        for args, ops in ref.items():
            assert ops.get("DMMA.8x8x4", 0) == 128 and _count(ops, "DMMA") == 128, (old, args)

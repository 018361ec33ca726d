"""The A^T (A x) kernels in the built library (cuobjdump -sass, no GPU needed): the row tiles arrive by bulk copy (UBLKCP) on
an mbarrier pipeline, every multiply and add is a separate DMUL / DADD (no DFMA, as in the reference's ddot and daxpy),
and nothing spills to local memory."""
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
        if "gm_tile_kernel" in mangled or "gm_fold_kernel" in mangled:
            res[mangled] = [m.group(1) for m in re.finditer(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Za-z0-9_.]*)[^;]*;", chunk)]
    return res


def _ops(kernels, name):
    found = {k: v for k, v in kernels.items() if name in k}
    assert len(found) == 1, list(kernels)
    return collections.Counter(op.split(".")[0] for op in next(iter(found.values())))


def test_tile_kernel_is_bulk_copy_fed_and_never_fuses(kernels):
    ops = _ops(kernels, "gm_tile_kernel")
    assert ops["UBLKCP"] >= 1 and ops["SYNCS"] >= 2
    assert ops["LDL"] == 0 and ops["STL"] == 0
    assert ops["DFMA"] == 0
    assert ops["DMUL"] >= 2 and ops["DADD"] >= 2


def test_fold_kernel_adds_separately(kernels):
    ops = _ops(kernels, "gm_fold_kernel")
    assert ops["DFMA"] == 0 and ops["DADD"] >= 1
    assert ops["LDL"] == 0 and ops["STL"] == 0

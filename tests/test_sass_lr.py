"""The logistic-regression kernels in the built library (cuobjdump -sass, no GPU needed): the row pieces arrive by bulk copy
(UBLKCP) on an mbarrier pipeline, every multiply and add of the margins and gradient sums is a separate DMUL / DADD (no
DFMA: the JVM never contracts), and nothing spills to local memory.  exp and the division of the sigmoid are built on DFMA;
they sit in an out-of-line subroutine after the kernel body, which is excluded from the DFMA check."""
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
        if "lr_grad_tile_kernel" in mangled or "lr_fold_kernel" in mangled:
            res[mangled] = [(int(m.group(1), 16), m.group(2), m.group(3)) for m in
                            re.finditer(r"/\*([0-9a-f]{4,})\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Za-z0-9_.]*)([^;]*);", chunk)]
    return res


def _ops(instrs):
    return collections.Counter(op.split(".")[0] for _, op, _ in instrs)


def test_lr_tile_kernel_is_bulk_copy_fed_and_never_fuses(kernels):
    tile = {k: v for k, v in kernels.items() if "lr_grad_tile_kernel" in k}
    assert len(tile) == 1
    instrs = next(iter(tile.values()))
    everything = _ops(instrs)
    assert everything["UBLKCP"] >= 1 and everything["SYNCS"] >= 2          # bulk copies completing on mbarriers
    assert everything["LDL"] == 0 and everything["STL"] == 0
    # the kernel body ends where the first called subroutine begins (integer division helpers, the sigmoid)
    targets = [int(m.group(1), 16) for _, op, rest in instrs if op.startswith("CALL") for m in [re.search(r"0x([0-9a-f]+)", rest)] if m]
    assert targets, "the sigmoid is expected out of line"
    body = _ops([i for i in instrs if i[0] < min(targets)])
    assert body["DFMA"] == 0
    assert body["DMUL"] >= 2 and body["DADD"] >= 2


def test_lr_fold_kernel_adds_and_multiplies_separately(kernels):
    fold = {k: v for k, v in kernels.items() if "lr_fold_kernel" in k}
    assert len(fold) == 1
    ops = _ops(next(iter(fold.values())))
    assert ops["DFMA"] == 0 and ops["DMUL"] >= 1 and ops["DADD"] >= 1
    assert ops["LDL"] == 0 and ops["STL"] == 0

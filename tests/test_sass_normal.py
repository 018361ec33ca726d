"""The StandardNormalGenerator kernels in the built library (cuobjdump -sass, no GPU needed): the count kernel has no DFMA
at all; in the write kernel every DFMA belongs to the correctly rounded divisions and the square root, which sit in the
out-of-line subroutines div_rn and polar_multiplier after the kernel body (a CALL marks where the body ends), so the body
itself has none; nothing spills to local memory."""
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
        for name in ("normal_count_kernel", "normal_write_kernel", "normal_scan_kernel"):
            if name in mangled:
                res[name] = [(int(m.group(1), 16), m.group(2), m.group(3)) for m in
                             re.finditer(r"/\*([0-9a-f]{4,})\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Za-z0-9_.]*)([^;]*);", chunk)]
    return res


def _ops(instrs):
    return collections.Counter(op.split(".")[0] for _, op, _ in instrs)


def test_all_three_kernels_are_built(kernels):
    assert set(kernels) == {"normal_count_kernel", "normal_write_kernel", "normal_scan_kernel"}


def test_count_kernel_never_fuses(kernels):
    ops = _ops(kernels["normal_count_kernel"])
    assert ops["DFMA"] == 0
    assert ops["DMUL"] >= 2 and ops["DADD"] >= 3                # two squares, their sum, two exact conversions
    assert ops["LDL"] == 0 and ops["STL"] == 0


def test_write_kernel_fuses_only_inside_division_and_square_root(kernels):
    instrs = kernels["normal_write_kernel"]
    ops = _ops(instrs)
    assert ops["LDL"] == 0 and ops["STL"] == 0
    targets = [int(m.group(1), 16) for _, op, rest in instrs if op.startswith("CALL") for m in [re.search(r"0x([0-9a-f]+)", rest)] if m]
    assert targets, "the division and the square root are expected out of line"
    body = _ops([i for i in instrs if i[0] < min(targets)])
    tail = [i for i in instrs if i[0] >= min(targets)]
    assert body["DFMA"] == 0
    assert body["DMUL"] >= 20 and body["DADD"] >= 10             # the polar step, fdlibm's log and the scaling
    tail_ops = _ops(tail)
    assert tail_ops["DFMA"] >= 1
    mufu = {op for _, op, _ in tail if op.startswith("MUFU")}
    assert {"MUFU.RCP64H", "MUFU.RSQ64H"} <= mufu, mufu          # the reciprocal and square-root seeds


def test_scan_kernel_does_not_spill(kernels):
    ops = _ops(kernels["normal_scan_kernel"])
    assert ops["LDL"] == 0 and ops["STL"] == 0

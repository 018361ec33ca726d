"""The NeuralNetwork kernels in the built library (cuobjdump -sass, no GPU needed): the fused backprop kernel is fed by bulk
copies (UBLKCP) on an mbarrier pipeline, spills nothing to local memory and, like the update kernel, sums without 64-bit
floating-point atomics or reductions, which is what makes a run repeat bit for bit."""
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
        if "nn_backprop_kernel" in mangled or "nn_apply_kernel" in mangled:
            res[mangled] = [m.group(1) for m in re.finditer(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Za-z0-9_.]*)[^;]*;", chunk)]
    return res


def _one(kernels, name):
    hit = [v for k, v in kernels.items() if name in k]
    assert len(hit) == 1, sorted(kernels)
    return hit[0], collections.Counter(op.split(".")[0] for op in hit[0])


def test_backprop_kernel_is_bulk_copy_fed_without_spills_or_atomics(kernels):
    instrs, ops = _one(kernels, "nn_backprop_kernel")
    assert ops["UBLKCP"] >= 1 and ops["SYNCS"] >= 2            # bulk copies completing on mbarriers
    assert ops["LDL"] == 0 and ops["STL"] == 0
    assert not [op for op in instrs if op.split(".")[0] in ("RED", "ATOM", "ATOMG", "ATOMS")]
    assert ops["DFMA"] >= 10 and ops["CALL"] >= 2              # the products; the sigmoid stays one out-of-line function


def test_apply_kernel_rounds_every_step_and_has_no_atomics(kernels):
    instrs, ops = _one(kernels, "nn_apply_kernel")
    assert ops["DFMA"] == 0 and ops["DMUL"] >= 1 and ops["DADD"] >= 2
    assert ops["LDL"] == 0 and ops["STL"] == 0
    assert not [op for op in instrs if op.split(".")[0] in ("RED", "ATOM", "ATOMG", "ATOMS")]

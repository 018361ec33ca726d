"""The matrix-file writer's kernels in the built library (cuobjdump -sass, no GPU needed): both are built, neither spills to
local memory, and the digits come from integer arithmetic alone: no DADD, DMUL, DFMA or MUFU (which would also be the
reciprocal behind a division by a run-time value)."""
import pytest

from tests.harness import count, family, ops

KERNELS = ("text_length_kernel", "text_write_kernel")


@pytest.mark.parametrize("name", KERNELS)
def test_kernel_is_built_and_does_not_spill(name):
    (instrs,) = family(name).values()
    c = ops(instrs)
    assert count(c, "LDL") == 0 and count(c, "STL") == 0


@pytest.mark.parametrize("name", KERNELS)
def test_digits_use_no_floating_point(name):
    (instrs,) = family(name).values()
    c = ops(instrs)
    for op in ("DADD", "DMUL", "DFMA", "MUFU"):
        assert count(c, op) == 0, op
    assert count(c, "IMAD") > 0                          # the 64 x 64 -> 128 products


def test_tables_are_read_from_shared_memory():
    (instrs,) = family("text_write_kernel").values()
    assert count(ops(instrs), "LDS") > 0
    assert count(ops(instrs), "LDC") < 64                # kernel parameters only: no table in the constant bank

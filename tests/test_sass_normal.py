"""The StandardNormalGenerator kernels in the built library (cuobjdump -sass, no GPU needed): the count kernel has no DFMA
at all; in the write kernel every DFMA belongs to the correctly rounded divisions and the square root, which sit in the
out-of-line subroutines div_rn and polar_multiplier after the kernel body (a CALL marks where the body ends), so the body
itself has none; nothing spills to local memory."""
from tests.harness import body, count, family, ops


def test_all_three_kernels_are_built():
    for name in ("normal_count_kernel", "normal_write_kernel", "normal_scan_kernel"):
        assert family(name)


def test_count_kernel_never_fuses():
    (instrs,) = family("normal_count_kernel").values()
    c = ops(instrs)
    assert count(c, "DFMA") == 0
    assert count(c, "DMUL") >= 2 and count(c, "DADD") >= 3                # two squares, their sum, two exact conversions
    assert count(c, "LDL") == 0 and count(c, "STL") == 0


def test_write_kernel_fuses_only_inside_division_and_square_root():
    (instrs,) = family("normal_write_kernel").values()
    c = ops(instrs)
    assert count(c, "LDL") == 0 and count(c, "STL") == 0
    head = body(instrs)
    tail = instrs[len(head):]                                               # the subroutines, in address order
    b = ops(head)
    assert count(b, "DFMA") == 0
    assert count(b, "DMUL") >= 20 and count(b, "DADD") >= 10               # the polar step, fdlibm's log and the scaling
    assert count(ops(tail), "DFMA") >= 1
    mufu = {op for _, op, _ in tail if op.startswith("MUFU")}
    assert {"MUFU.RCP64H", "MUFU.RSQ64H"} <= mufu, mufu                     # the reciprocal and square-root seeds


def test_scan_kernel_does_not_spill():
    (instrs,) = family("normal_scan_kernel").values()
    c = ops(instrs)
    assert count(c, "LDL") == 0 and count(c, "STL") == 0

"""The logistic-regression kernels in the built library (cuobjdump -sass, no GPU needed): the row pieces arrive by bulk copy
(UBLKCP) on an mbarrier pipeline, every multiply and add of the margins and gradient sums is a separate DMUL / DADD (no
DFMA: the JVM never contracts), and nothing spills to local memory.  exp and the division of the sigmoid are built on DFMA;
they sit in an out-of-line subroutine after the kernel body, which is excluded from the DFMA check."""
from tests.harness import body, count, family, ops


def test_lr_tile_kernel_is_bulk_copy_fed_and_never_fuses():
    tile = family("lr_grad_tile_kernel")
    assert len(tile) == 1
    instrs = next(iter(tile.values()))
    everything = ops(instrs)
    assert count(everything, "UBLKCP") >= 1 and count(everything, "SYNCS") >= 2       # bulk copies completing on mbarriers
    assert count(everything, "LDL") == 0 and count(everything, "STL") == 0
    # the kernel body ends where the first called subroutine begins (integer division helpers, the sigmoid)
    b = ops(body(instrs))
    assert count(b, "DFMA") == 0
    assert count(b, "DMUL") >= 2 and count(b, "DADD") >= 2


def test_lr_fold_kernel_adds_and_multiplies_separately():
    fold = family("lr_fold_kernel")
    assert len(fold) == 1
    c = ops(next(iter(fold.values())))
    assert count(c, "DFMA") == 0 and count(c, "DMUL") >= 1 and count(c, "DADD") >= 1
    assert count(c, "LDL") == 0 and count(c, "STL") == 0

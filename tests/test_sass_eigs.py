"""The A^T (A x) kernels in the built library (cuobjdump -sass, no GPU needed): the row tiles arrive by bulk copy (UBLKCP) on
an mbarrier pipeline, every multiply and add is a separate DMUL / DADD (no DFMA, as in the reference's ddot and daxpy),
and nothing spills to local memory."""
from tests.harness import count, family, ops


def test_tile_kernel_is_bulk_copy_fed_and_never_fuses():
    fam = family("gm_tile_kernel")
    assert len(fam) == 1, list(fam)
    c = ops(next(iter(fam.values())))
    assert count(c, "UBLKCP") >= 1 and count(c, "SYNCS") >= 2
    assert count(c, "LDL") == 0 and count(c, "STL") == 0
    assert count(c, "DFMA") == 0
    assert count(c, "DMUL") >= 2 and count(c, "DADD") >= 2


def test_fold_kernel_adds_separately():
    fam = family("gm_fold_kernel")
    assert len(fam) == 1, list(fam)
    c = ops(next(iter(fam.values())))
    assert count(c, "DFMA") == 0 and count(c, "DADD") >= 1
    assert count(c, "LDL") == 0 and count(c, "STL") == 0

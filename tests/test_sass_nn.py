"""The NeuralNetwork kernels in the built library (cuobjdump -sass, no GPU needed): the fused backprop kernel is fed by bulk
copies (UBLKCP) on an mbarrier pipeline, spills nothing to local memory and, like the update kernel, sums without 64-bit
floating-point atomics or reductions, which is what makes a run repeat bit for bit."""
from tests.harness import count, family, ops

ATOMICS = ("RED", "ATOM", "ATOMG", "ATOMS")


def test_backprop_kernel_is_bulk_copy_fed_without_spills_or_atomics():
    fam = family("nn_backprop_kernel")
    assert len(fam) == 1, sorted(fam)
    c = ops(next(iter(fam.values())))
    assert count(c, "UBLKCP") >= 1 and count(c, "SYNCS") >= 2            # bulk copies completing on mbarriers
    assert count(c, "LDL") == 0 and count(c, "STL") == 0
    assert not [op for op in c if op.split(".")[0] in ATOMICS]
    assert count(c, "DFMA") >= 10 and count(c, "CALL") >= 2              # the products; the sigmoid stays one out-of-line function


def test_apply_kernel_rounds_every_step_and_has_no_atomics():
    fam = family("nn_apply_kernel")
    assert len(fam) == 1, sorted(fam)
    c = ops(next(iter(fam.values())))
    assert count(c, "DFMA") == 0 and count(c, "DMUL") >= 1 and count(c, "DADD") >= 2
    assert count(c, "LDL") == 0 and count(c, "STL") == 0
    assert not [op for op in c if op.split(".")[0] in ATOMICS]

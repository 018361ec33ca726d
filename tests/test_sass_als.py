"""The ALS kernels in the built library (cuobjdump -sass, no GPU needed): the assembly-only instances of als_kernel add and
multiply with separate DADD / DMUL (no DFMA: the JVM never contracts), and no instance touches local memory."""
from tests.harness import count, family, ops

ALS = "2mb10als_kernelI"                                       # mb::als_kernel<...>


def test_assembly_instances_never_fuse():
    # als_kernel<G, EPT, SOLVE = false>: the mangled template argument list ends in Lb0E
    asm = {k: ops(v) for k, v in family(ALS).items() if "Lb0E" in k}
    assert len(asm) == 5, sorted(family(ALS))          # one per rank bucket
    for c in asm.values():
        assert count(c, "DFMA") == 0
        assert count(c, "DMUL") >= 2 and count(c, "DADD") >= 2


def test_no_local_memory():
    kernels = family(ALS)
    assert len(kernels) == 10
    for instrs in kernels.values():
        c = ops(instrs)
        assert count(c, "LDL") == 0 and count(c, "STL") == 0

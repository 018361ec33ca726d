"""The PageRank kernels in the built library (cuobjdump -sass, no GPU needed): every instance of pagerank_step_kernel
multiplies and adds in fp64 with separate DMUL and DADD (no DFMA: the JVM never contracts a * b + c), and no PageRank
kernel touches local memory."""
from tests.harness import count, family, ops


def test_step_kernels_multiply_and_add_separately():
    kernels = family("pagerank_cu")
    steps = [ops(v) for k, v in kernels.items() if "pagerank_step_kernel" in k]
    assert len(steps) == 2, sorted(kernels)                 # the light-row and the heavy-row instance
    for c in steps:
        assert count(c, "DFMA") == 0
        assert count(c, "DMUL") >= 1 and count(c, "DADD") >= 1


def test_no_local_memory():
    kernels = family("pagerank_cu")
    assert len(kernels) == 3, sorted(kernels)
    for instrs in kernels.values():
        c = ops(instrs)
        assert count(c, "LDL") == 0 and count(c, "STL") == 0

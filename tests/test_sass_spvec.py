"""The SparseVecMatrix kernels in the built library (cuobjdump -sass, no GPU needed): the product kernels multiply and add
in float32 with separate FMUL and FADD (no FFMA: the JVM never contracts a * b + c), and no spvec kernel touches local
memory."""
import pytest

from tests.harness import count, family, ops

PRODUCT_KERNELS = ("spvec_warp_kernelILb1E", "spvec_cta_kernelILb1E", "spvec_window_kernelILb1E")


@pytest.mark.parametrize("needle", PRODUCT_KERNELS)
def test_products_multiply_and_add_separately(needle):
    kernels = family("spvec_cu")
    fam = [ops(v) for k, v in kernels.items() if needle in k]
    assert len(fam) == 1, (needle, sorted(kernels))
    c = fam[0]
    assert count(c, "FFMA") == 0
    assert count(c, "FMUL") >= 1 and count(c, "FADD") >= 1


def test_no_local_memory():
    kernels = family("spvec_cu")
    assert len(kernels) == 11, sorted(kernels)
    for instrs in kernels.values():
        c = ops(instrs)
        assert count(c, "LDL") == 0 and count(c, "STL") == 0

"""The sparse kernels in the built library (cuobjdump -sass, no GPU needed): no fused multiply-add anywhere (the results
are bit-identical to the reference loops only with separate DMUL and DADD), and no spills to local memory."""
import pytest

from tests.harness import count, family, ops

SPARSE_KERNELS = ("csc_to_dense_kernel", "dense_sparse_kernel", "sparse_dense_kernel", "spgemm_kernel", "csr_count_kernel",
                  "scan_inplace_kernel", "csr_scatter_kernel", "csr_sort_kernel", "sample_rows_kernel")


@pytest.mark.parametrize("needle", SPARSE_KERNELS)
def test_sparse_kernel_has_no_dfma_and_no_spills(needle):
    fam = {k: v for k, v in family("sparse_cu").items() if needle in k}
    assert len(fam) == 1, (needle, list(fam))
    c = ops(next(iter(fam.values())))
    assert count(c, "DFMA") == 0
    assert count(c, "LDL") == 0 and count(c, "STL") == 0


@pytest.mark.parametrize("needle", ["dense_sparse_kernel", "sparse_dense_kernel", "spgemm_kernel"])
def test_products_multiply_and_add_separately(needle):
    c = ops(next(v for k, v in family("sparse_cu").items() if needle in k))
    assert count(c, "DMUL") >= 1 and count(c, "DADD") >= 1

"""The sparse kernels in the built library (cuobjdump -sass, no GPU needed): no fused multiply-add anywhere (the results
are bit-identical to the reference loops only with separate DMUL and DADD), and no spills to local memory."""
import collections
import re
import shutil
import subprocess

import pytest

from marlin_b200 import _native as nat

SPARSE_KERNELS = ("csc_to_dense_kernel", "dense_sparse_kernel", "sparse_dense_kernel", "spgemm_kernel", "csr_count_kernel",
                  "scan_inplace_kernel", "csr_scatter_kernel", "csr_sort_kernel", "sample_rows_kernel")


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
        res[mangled] = collections.Counter(m.group(1) for m in re.finditer(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Za-z0-9_.]*)", chunk))
    return res


def _count(ops, prefix):
    return sum(v for k, v in ops.items() if k.split(".")[0] == prefix)


@pytest.mark.parametrize("needle", SPARSE_KERNELS)
def test_sparse_kernel_has_no_dfma_and_no_spills(kernels, needle):
    fam = {k: v for k, v in kernels.items() if needle in k and "sparse_cu" in k}
    assert len(fam) == 1, (needle, list(fam))
    ops = next(iter(fam.values()))
    assert _count(ops, "DFMA") == 0
    assert _count(ops, "LDL") == 0 and _count(ops, "STL") == 0


@pytest.mark.parametrize("needle", ["dense_sparse_kernel", "sparse_dense_kernel", "spgemm_kernel"])
def test_products_multiply_and_add_separately(kernels, needle):
    ops = next(v for k, v in kernels.items() if needle in k and "sparse_cu" in k)
    assert _count(ops, "DMUL") >= 1 and _count(ops, "DADD") >= 1

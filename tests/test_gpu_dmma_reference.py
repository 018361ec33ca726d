"""The m16n8k4 fp64 kernels against their m8n8k4 reference instances (mb_set_dmma_reference), bit for bit.

m16n8k4 is two m8n8k4 stacked in M that share the B fragment, and the kernels pair m-tiles without changing which k
values reach an element or in which order, so every entry point that runs the DMMA mainloop must give identical bits on
either shape.  Each case also checks with torch.profiler which kernels ran: the default path runs the *dmma16x8* kernels
and the reference path runs the older names and nothing else, so the equality compares two different kernels."""
import ctypes as C

import pytest

from marlin_b200 import _native as nat

pytestmark = pytest.mark.gpu

REFERENCE = ("gemm_f64_dmma_kernel", "gemm_f64_dmma_grouped_kernel", "syrk_f64_dmma_kernel")


@pytest.fixture(scope="module")
def rt():
    import marlin_b200 as mb
    r = mb.Runtime.get()
    r.set_dmma_reference(False)
    yield r
    r.set_dmma_reference(False)


def _run(rt, reference, fn):
    """fn() with the reference kernels on or off; returns (its result, the names of the CUDA kernels it ran).  A trace
    with no GPU activity at all is a capture the profiler missed (every fn here launches kernels), so fn runs again, at
    most twice more; its result does not depend on the attempt."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    rt.set_dmma_reference(reference)
    try:
        for _ in range(3):
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                out = fn()
                torch.cuda.synchronize()
            names = {e.name for e in prof.events() if e.device_type.name == "CUDA"}
            if names:
                break
    finally:
        rt.set_dmma_reference(False)
    return out, names


def check_same(rt, fn, family):
    """fn() returns a list of fp64 tensors; they must be bitwise equal on both shapes, and the DMMA kernel of `family`
    ('gemm', 'grouped' or 'syrk') must be the one that ran on each."""
    import torch
    new, new_names = _run(rt, False, fn)
    ref, ref_names = _run(rt, True, fn)
    full = {"gemm": "gemm_f64_dmma16x8_kernel", "grouped": "gemm_f64_dmma16x8_grouped_kernel", "syrk": "syrk_f64_dmma16x8_kernel"}[family]
    old = {"gemm": "gemm_f64_dmma_kernel", "grouped": "gemm_f64_dmma_grouped_kernel", "syrk": "syrk_f64_dmma_kernel"}[family]
    assert any(full in n for n in new_names), sorted(new_names)
    assert not any(r in n for n in new_names for r in REFERENCE), sorted(new_names)
    assert any(old in n for n in ref_names), sorted(ref_names)
    assert not any("dmma16x8" in n for n in ref_names), sorted(ref_names)
    assert len(new) == len(ref)
    for a, b in zip(new, ref):
        assert a.dtype == torch.float64 and a.shape == b.shape
        if not torch.equal(a.view(torch.int64), b.view(torch.int64)):
            diff = (a - b).abs()
            raise AssertionError(f"m16n8k4 differs from m8n8k4: {int((diff != 0).sum())} elements, max |diff| {float(diff.max())}")


def _randn(gen, n):
    import torch
    return torch.randn(n, generator=gen, device="cuda", dtype=torch.float64)


@pytest.mark.parametrize("m, n, k", [(129, 257, 4099), (1000, 1000, 1000), (4096, 4096, 4096)])
@pytest.mark.parametrize("ta", [0, 1])
@pytest.mark.parametrize("tb", [0, 1])
@pytest.mark.parametrize("beta", [0.0, 1.0])
def test_dgemm_device(rt, m, n, k, ta, tb, beta):
    """Leading dimensions are rounded up to even so that odd sizes still run the TMA kernels, not the CUDA-core one."""
    import torch
    gen = torch.Generator(device="cuda").manual_seed(1000 * ta + 100 * tb + int(beta) + m)
    even = lambda x: (x + 1) & ~1                                                   # noqa: E731
    lda, ldb, ldc = even(k if ta else m), even(n if tb else k), even(m)
    A, B, C0 = _randn(gen, lda * (m if ta else k)), _randn(gen, ldb * (k if tb else n)), _randn(gen, ldc * n)

    def fn():
        rt.sync_stream()
        Cd = C0.clone()
        nat.check(rt.lib.mb_dgemm_device(rt.ctx, b"T" if ta else b"N", b"T" if tb else b"N", m, n, k, 0.75,
                                         C.c_void_p(A.data_ptr()), lda, C.c_void_p(B.data_ptr()), ldb, beta,
                                         C.c_void_p(Cd.data_ptr()), ldc))
        return [Cd]

    check_same(rt, fn, "gemm")


@pytest.mark.parametrize("shape", ["ragged3x3x3", "headline2x2"])
def test_matmul_blocked(rt, shape):
    import marlin_b200 as mb
    if shape == "ragged3x3x3":
        # blocks of 334 / 332 rows, 434 / 432 k and 300 columns: ragged against the 128-wide tiles, and all of even
        # length, so that every block stays TMA-addressable and the whole multiply is one grouped launch
        A = mb.MTUtils.randomBlockMatrix(None, 1000, 1300, 3, 3, seed=42)
        B = mb.MTUtils.randomBlockMatrix(None, 1300, 900, 3, 3, seed=43)
    else:
        A = mb.MTUtils.randomBlockMatrix(None, 16384, 16384, 2, 2, seed=42)     # the benchmark's multiply
        B = mb.MTUtils.randomBlockMatrix(None, 16384, 16384, 2, 2, seed=43)

    def fn():
        Cm = A.multiply(B)
        blocks = [s for _, s in sorted(Cm.blocks, key=lambda bs: (bs[0].row, bs[0].column))]
        assert len(blocks) == (9 if shape == "ragged3x3x3" else 4) and all(s.is_packed() for s in blocks)
        return [s.buf for s in blocks]

    check_same(rt, fn, "grouped")


def test_matmul_rowsharded(rt):
    import torch
    from marlin_b200.matrix.sub_matrix import SubMatrix
    rows, k, n = 131072, 1024, 1024
    gen = torch.Generator(device="cuda").manual_seed(7)
    A = SubMatrix(buf=_randn(gen, rows * k), rows=rows, cols=k, ld=k, is_transpose=True)      # row-major row shard
    B = SubMatrix(buf=_randn(gen, k * n), rows=k, cols=n, ld=k)

    def fn():
        rt.sync_stream()
        Cr = SubMatrix(buf=torch.empty(rows * n, device="cuda", dtype=torch.float64), rows=rows, cols=n, ld=n, is_transpose=True)
        nat.check(rt.lib.mb_matmul_rowsharded(rt.ctx, A.handle(), B.handle(), Cr.handle()))
        return [Cr.buf]

    check_same(rt, fn, "gemm")


@pytest.mark.parametrize("n, m", [(1024, 65536), (4096, 8192), (333, 20000)])
@pytest.mark.parametrize("form", ["rows", "columns"])
def test_gramian(rt, n, m, form):
    """rows: a row-major row shard (a transposed view; ld = n rounded up to even so that TMA can read it), G = X X^T on
    the array underneath; columns: a column-major m x n block, G = A^T A.  n = 1024 and 333 split K over partials."""
    import torch
    from marlin_b200.matrix.sub_matrix import SubMatrix
    gen = torch.Generator(device="cuda").manual_seed(n + m)
    if form == "rows":
        ld = (n + 1) & ~1
        A = SubMatrix(buf=_randn(gen, m * ld), rows=m, cols=n, ld=ld, is_transpose=True)
    else:
        A = SubMatrix(buf=_randn(gen, m * n), rows=m, cols=n, ld=m)
    if n < 4096:
        assert rt.lib.mb_gramian_workspace_bytes(n, m, torch.cuda.get_device_properties(0).multi_processor_count) > 0

    def fn():
        return [A.gramian().buf]

    check_same(rt, fn, "syrk")

"""The full-rate fp64 kernels in the built library (cuobjdump -sass, no GPU needed): every fp64 GEMM, grouped and Gramian
kernel that production launches issues DMMA.16x8x4 (mma.sync.m16n8k4, twice the fp64 rate of DMMA.8x8x4 on H100), fed by
the same TMA ring and the same 24 conflict-free LDS.128 per k16 slab as the m8n8k4 reference instances, without spills."""
import pytest

from tests.harness import count, ops, sass


@pytest.mark.parametrize("needle, instances", [("gemm_f64_dmma16x8_kernel", 4),           # the four N/T operand forms
                                               ("gemm_f64_dmma16x8_grouped_kernel", 1),   # the blocked multiply
                                               ("syrk_f64_dmma16x8_kernel", 2)])          # Gramian: (N,T) and (T,N)
def test_fp64_kernels_issue_dmma_16x8x4(needle, instances):
    fam = {k: ops(v) for k, v in sass().items() if needle in k}
    assert len(fam) == instances, sorted(fam)
    for name, c in fam.items():
        assert c.get("DMMA.16x8x4", 0) == 64, (name, c.get("DMMA.16x8x4"))       # one k16 slab of a 64x32 warp tile
        assert count(c, "DMMA") == 64, name                                       # ... and no other DMMA shape
        lds = sum(v for k, v in c.items() if k.startswith("LDS"))
        assert lds == 24 and all(k.startswith("LDS.128") or not k.startswith("LDS") for k in c), name
        assert count(c, "UTMALDG") >= 2 and count(c, "SYNCS") >= 10, name        # TMA loads + mbarrier pipeline
        assert count(c, "USETMAXREG") == 2, name                                  # producer gives registers to consumers
        assert count(c, "LDL") == 0 and count(c, "STL") == 0, name                # no spills


def test_reference_instances_are_the_same_kernels_at_m8n8k4():
    """Each full-rate kernel has its m8n8k4 reference instance (mb_set_dmma_reference) under the older name."""
    for old, new in (("gemm_f64_dmma_kernel", "gemm_f64_dmma16x8_kernel"),
                     ("gemm_f64_dmma_grouped_kernel", "gemm_f64_dmma16x8_grouped_kernel"),
                     ("syrk_f64_dmma_kernel", "syrk_f64_dmma16x8_kernel")):
        ref = {k.split(old, 1)[1]: ops(v) for k, v in sass().items() if old in k}
        full = {k.split(new, 1)[1]: v for k, v in sass().items() if new in k}
        assert ref and set(ref) == set(full), (old, sorted(ref), sorted(full))   # same template instances
        for args, c in ref.items():
            assert c.get("DMMA.8x8x4", 0) == 128 and count(c, "DMMA") == 128, (old, args)

"""The SVD kernels in the built library (cuobjdump -sass, no GPU needed): the Gramian runs the DMMA mainloop fed by TMA,
the reduce-and-mirror pass uses 128-bit accesses, and none of the new kernels spills to local memory."""
from tests.harness import count, family, ops


def test_gramian_is_dmma_fed_by_tma():
    fam = family("syrk_f64_dmma_kernel")
    assert len(fam) == 2                                       # row-shard (N,T) and column-major (T,N) operands
    for name, instrs in fam.items():
        c = ops(instrs)
        assert c.get("DMMA.8x8x4", 0) == 128, name
        assert count(c, "UTMALDG") >= 2 and count(c, "SYNCS") >= 10, name
        assert count(c, "LDL") == 0 and count(c, "STL") == 0, name


def test_svd_kernels_do_not_spill():
    for needle in ("gram_reduce_mirror_kernel", "jacobi_round_kernel", "jacobi_init_kernel", "jacobi_gather_kernel"):
        for name, instrs in family(needle).items():
            c = ops(instrs)
            assert count(c, "LDL") == 0 and count(c, "STL") == 0, name
    fam = family("gram_reduce_mirror_kernel")
    assert len(fam) == 2                                       # 128-bit or scalar reads of the partials
    for name, instrs in fam.items():
        c = ops(instrs)
        assert any(k.startswith("STG.E.128") for k in c), name
        if "ILb1E" in name:
            assert any(k.startswith("LDG.E.128") for k in c), name
    for name, instrs in family("jacobi_round_kernel").items():
        c = ops(instrs)
        assert any(k.startswith("LDG.E.128") for k in c) and any(k.startswith("STG.E.128") for k in c), name

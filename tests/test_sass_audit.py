"""What the built library actually contains (cuobjdump -sass of libmarlin_b200.so, no GPU needed): the hot kernels are
sm_90a code that uses the units the design says they use — DMMA.8x8x4 fed by TMA for fp64, warpgroup MMA (HGMMA / IGMMA,
the SASS of wgmma.mma_async) fed by TMA with register accumulators for bf16 and the int8 split — and no kernel spills
registers to local memory in its inner loop.  That every kernel is sm_90a code is asserted where the SASS is read
(tests/harness.py)."""
from tests.harness import count, family, ops


def test_fp64_gemm_is_dmma_fed_by_tma():
    fam = {**family("gemm_f64_dmma_kernel"), **family("gemm_f64_dmma_grouped_kernel")}
    assert len(fam) == 5                                       # four N/T instances + the grouped launch
    for name, instrs in fam.items():
        c = ops(instrs)
        assert c.get("DMMA.8x8x4", 0) == 128, (name, c.get("DMMA.8x8x4"))       # one k16 slab of a 64x32 warp tile
        assert count(c, "UTMALDG") >= 2 and count(c, "SYNCS") >= 10              # TMA loads + mbarrier pipeline
        assert count(c, "USETMAXREG") == 2                                        # producer gives registers to consumers
        assert count(c, "LDL") == 0 and count(c, "STL") == 0                      # no spills
        lds = sum(v for k, v in c.items() if k.startswith("LDS"))
        assert lds == 24 and all(k.startswith("LDS.128") or not k.startswith("LDS") for k in c)   # 24 conflict-free LDS.128 per slab


def test_bf16_and_int8_gemms_are_wgmma_fed_by_tma():
    bf = family("gemm_bf16_wgmma_kernel")
    assert len(bf) == 4
    for name, instrs in bf.items():
        c = ops(instrs)
        assert count(c, "HGMMA") >= 1 and count(c, "IGMMA") == 0                 # wgmma f32 += bf16 x bf16
        assert count(c, "WARPGROUP") >= 1 and count(c, "UTMALDG") >= 2 and count(c, "SYNCS") >= 1
        assert count(c, "HMMA") == 0                                              # no mma.sync fallback
        assert count(c, "LDL") == 0 and count(c, "STL") == 0                      # accumulator stays in registers
    i8 = family("gemm_ozaki_i8")
    assert len(i8) == 1
    for name, instrs in i8.items():
        c = ops(instrs)
        assert count(c, "IGMMA") >= 1 and count(c, "HGMMA") == 0                 # wgmma s32 += s8 x s8
        assert count(c, "WARPGROUP") >= 1 and count(c, "UTMALDG") >= 2 and count(c, "IMMA") == 0
        assert count(c, "LDL") == 0 and count(c, "STL") == 0


def test_hbm_kernels_use_128_bit_accesses_and_do_not_spill():
    for needle, ld, st in (("binary_flat_kernel", "LDG.E.128", "STG.E.128"), ("unary_flat_kernel", "LDG.E.128", "STG.E.128"),
                           ("transpose_f64_tile_kernel", "LDG.E.128", "STG.E.128"), ("gemv_n_kernel", "LDG.E.128", None),
                           ("gemv_t_kernel", "LDG.E.128", None), ("ger_kernel", None, "STG.E.128"),
                           ("fill_uniform_kernel", None, "STG.E.128")):
        for name, instrs in family(needle).items():
            c = ops(instrs)
            if "unary_flat_kernelILi14" in name:
                ld_ok = True                                    # EW_FILL reads nothing
            else:
                ld_ok = ld is None or any(k.startswith(ld) for k in c)
            assert ld_ok, (name, [k for k in c if k.startswith("LDG")])
            assert st is None or any(k.startswith(st) for k in c), (name, [k for k in c if k.startswith("STG")])
            assert count(c, "LDL") == 0 and count(c, "STL") == 0, name

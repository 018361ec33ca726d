"""One process with MARLIN_B200_BF16_KCHAIN set (the library reads the cap once): the K-chain split of fp32 bf16 products
on exact integer data, through mb_matmul_blocked_subset and mb_block_gemm, with its launch counts; with the cap off (0)
also the accuracy at total K = 65536.  Prints one JSON line."""
import ctypes as C
import json
import os
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from marlin_b200 import _native as nat                                      # noqa: E402
from tests import test_gpu_bf16_exact as t                                  # noqa: E402

# (rows, K per tile, cols).  cap 96: pieces shorter than a tile, their K tails zero-filled by the TMA inside a segment;
# cap 1000: cuts at offsets that are multiples of 8 but not of 64; cap 100: cuts at offsets that break 16-byte
# alignment (those pieces of B are staged); cap 0: one chain.
GRIDS = [([136], [4000] * 3, [264]), ([64], [1104] * 8, [40]), ([200], [72, 136, 130, 8], [264]), ([37], [333, 96], [21])]


def main():
    cap = int(os.environ["MARLIN_B200_BF16_KCHAIN"])
    lib = nat.load()
    ctx = nat.c_ctx()
    nat.check(lib.mb_init(0, C.byref(ctx)))
    gpu = (lib, ctx)
    cases = 0
    for g, (rows, Ks, cols) in enumerate(GRIDS):
        got, ref, n_launch, clean = t.blocked(gpu, rows, Ks, cols, nat.MB_F32, seed=50 + g)
        assert np.array_equal(got[(0, 0)], ref[(0, 0)]) and clean[(0, 0)], (cap, g)
        want = t.chain_launches(Ks, cap, rows[0])
        assert n_launch == want, (cap, g, n_launch, want)
        # one block GEMM over the whole K: pieces of one segment, with and without accumulate
        rng = np.random.default_rng(60 + g)
        A, B = t.ints(rng, (rows[0], sum(Ks))), t.ints(rng, (sum(Ks), cols[0]))
        for C0 in (None, t.ints(rng, (rows[0], cols[0]), 1000)):
            c, ok, n1 = t.block_gemm(gpu, A, B, 0, 0, nat.MB_F32, C0=C0)
            assert np.array_equal(c, t.expected(A, B, nat.MB_F32, C0)) and ok, (cap, g, C0 is not None)
            want = t.chain_launches([sum(Ks)], cap, t.ld_for(rows[0], "aligned")[0], b_ld=t.ld_for(sum(Ks), "aligned")[0])
            assert n1 == want, (cap, g, n1, want)
        c, ok, _ = t.block_gemm(gpu, A, B, 1, 1, nat.MB_F32, layout="odd")   # transposed, staged operands
        assert np.array_equal(c, t.expected(A, B, nat.MB_F32)) and ok, (cap, g)
        cases += 1
    errors = t.accuracy_errors(gpu) if cap == 0 else {}
    lib.mb_shutdown(ctx)
    print(json.dumps({"cap": cap, "cases": cases, "errors": errors}))


if __name__ == "__main__":
    main()

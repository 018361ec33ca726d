"""The bf16 wgmma GEMM on exact integer data, across tiles, waves, K chains, views and degenerate shapes.

The key fact: with bf16 operands that are small integers (|a|, |b| <= 4, exact in bf16) every product is exact in fp32
and every partial sum is an integer of magnitude <= 16 K <= 2^20 for K <= 65536.  So, as long as the tensor core keeps at
least 21 significant bits aligned to the largest addend, the fp32 result is exact in ANY summation order, tiling, chain
split or truncation mode: an fp32 C must equal the fp64 host product, and a bf16 C must equal that product (plus the
old C under accumulate) rounded to nearest-even once.  Every assertion on integer data below is therefore array_equal.

Random (non-integer) data is used only where a result is compared with the same call on other operands (views against
packed copies: bit-identical, because staging copies values and changes no summation) and for the accuracy at
config-5 chain length (K = 65536), which is checked against the documented tolerance of 1e-4 per element.
"""
import ctypes as C
import json
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from marlin_b200 import _native as nat
from tests.harness import gpu  # noqa: F401  (a fixture)
from tests.test_gpu_fp64_edges import bf16_rne

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
KCHAIN_DEFAULT = 8192


# ------------------------------------------------------------------------------------------------------------ helpers
def torch_dtype(dt):
    import torch
    return {nat.MB_BF16: torch.bfloat16, nat.MB_F32: torch.float32, nat.MB_F64: torch.float64}[dt]


def bf16_round(x):
    """Round-to-nearest-even to 8 significant bits on the fp64 bit pattern (vectorised; for finite values inside bf16's
    normal range, which is all the integer data here holds).  Pinned against bf16_rne in test_bf16_round_matches_rne."""
    x = np.ascontiguousarray(x, dtype=np.float64)
    b = x.view(np.uint64)
    lsb = (b >> np.uint64(45)) & np.uint64(1)
    r = (b + np.uint64((1 << 44) - 1) + lsb) & ~np.uint64((1 << 45) - 1)
    return r.view(np.float64)


def ints(rng, shape, lim=4):
    return rng.integers(-lim, lim + 1, size=shape).astype(np.float64)


def to_bf16_values(x):
    """The bf16 values nearest x (as fp64): inputs for the tests on random data, so that storing them is exact."""
    import torch
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float64)).to(torch.bfloat16).to(torch.float64).numpy()


class Stored:
    """A rows x cols matrix stored column-major with leading dimension `ld` at element `offset` of a flat device tensor
    whose every other element holds `fill` (NaN: a read outside the view poisons the result)."""

    def __init__(self, x, dtype, ld=None, offset=0, fill=np.nan, pad=64):
        import torch
        x = np.asarray(x, dtype=np.float64)
        self.rows, self.cols = x.shape
        self.ld = ld if ld is not None else max(1, self.rows)
        self.offset, self.dtype, self.fill = offset, dtype, fill
        flat = np.full(offset + self.ld * self.cols + pad, fill, dtype=np.float64)
        self._window(flat)[:] = x
        self.t = torch.from_numpy(flat).to(torch_dtype(dtype)).cuda()
        torch.cuda.synchronize()

    def _window(self, flat):
        """The rows x cols matrix as a strided view of the flat column-major array."""
        return flat[self.offset:self.offset + self.ld * self.cols].reshape(self.cols, self.ld)[:, :self.rows].T

    def flat(self):
        import torch
        return self.t.to(torch.float64).cpu().numpy()

    def values(self):
        return self.read()[0]

    def untouched_outside(self):
        return self.read()[1]

    def read(self):
        """(the matrix, whether every element outside it still holds the fill value bit for bit, NaN == NaN)."""
        f = self.flat()
        vals = np.array(self._window(f))
        self._window(f)[:] = self.fill
        return vals, bool(np.all(np.isnan(f))) if np.isnan(self.fill) else bool(np.all(f == self.fill))

    def block(self, gpu, trans=False):
        """The block over the stored matrix; trans: its transpose view (mb_block_view_t)."""
        lib, ctx = gpu
        h = nat.c_blk()
        nat.check(lib.mb_block_wrap(ctx, C.c_void_p(self.t.data_ptr()), self.offset, self.rows, self.cols, self.ld, 0,
                                    self.dtype, C.byref(h)))
        if not trans:
            return h
        v = nat.c_blk()
        nat.check(lib.mb_block_view_t(ctx, h, C.byref(v)))
        lib.mb_block_free(ctx, h)
        return v


def ld_for(rows, layout):
    """'aligned': ld a multiple of 8, base at element 0 (the TMA reads the operand in place); 'odd': ld = rows + 1 and
    base at element 3, 6 bytes past 16-byte alignment (the operand is staged first)."""
    if layout == "aligned":
        return max(8, -(-rows // 8) * 8), 0
    return rows + 1 if (rows + 1) % 8 else rows + 2, 3


def operand(x, trans, layout, fill=np.nan):
    """Logical operand x stored as x (trans=False) or as x^T (trans=True), in bf16."""
    s = x.T if trans else x
    ld, off = ld_for(s.shape[0], layout)
    return Stored(s, nat.MB_BF16, ld=ld, offset=off, fill=fill)


def launches(gpu):
    return gpu[0].mb_launch_count(gpu[1])


def sync(gpu):
    nat.check(gpu[0].mb_synchronize(gpu[1]))


def block_gemm(gpu, A, B, ta, tb, cdt, C0=None, ct=False, layout="aligned", fill=np.nan):
    """C = op(A) op(B) (+ C0 under accumulate) through mb_block_gemm with A, B given logically; ct: C is the transpose
    view of a row-major array (the swapped call C^T = B^T A^T).  Returns (C values, whether C's parent is untouched
    outside C, GEMM launches)."""
    lib, ctx = gpu
    m, n = A.shape[0], B.shape[1]
    sa, sb = operand(A, ta, layout), operand(B, tb, layout)
    start = np.full((m, n), np.nan) if C0 is None else C0
    cst = start.T if ct else start
    ld, off = ld_for(cst.shape[0], layout)
    sc = Stored(cst, cdt, ld=ld, offset=off + (1 if layout == "odd" else 0), fill=fill)
    ha, hb, hc = sa.block(gpu, ta), sb.block(gpu, tb), sc.block(gpu, ct)
    l0 = launches(gpu)
    nat.check(lib.mb_block_gemm(ctx, ha, hb, hc, int(C0 is not None)))
    sync(gpu)
    n_launch = launches(gpu) - l0
    for h in (ha, hb, hc):
        lib.mb_block_free(ctx, h)
    got, clean = sc.read()
    return (got.T if ct else got), clean, n_launch


def expected(A, B, cdt, C0=None):
    ref = A @ B + (0.0 if C0 is None else C0)
    return ref if cdt == nat.MB_F32 else bf16_round(ref)


def chain_launches(Ks, cap, a_ld, c_f32=True, b_ld=None, max_seg=8):
    """Launches (GEMMs + operand copies) of one C block on the segment path, restated from the library's rule: an fp32 C
    is built from pieces of at most `cap` k (0 = unlimited) and 8 pieces per launch, a bf16 C from one launch.  A(kk) is
    stored with ld = a_ld and B(kk) with ld = b_ld (default K_kk), each 16-byte aligned; a piece's operand is copied when
    its first element is not 16-byte aligned or its ld % 8 != 0 (A: columns k0.. -> offset k0 * ld; B: rows k0.. -> k0)."""
    cap = cap if (c_f32 and cap > 0) else 1 << 62
    total, in_group, npieces, copies = 0, 0, 0, 0
    for K in Ks:
        k0 = 0
        while k0 < K:
            ln = min(K - k0, cap - in_group)
            copies += int(a_ld % 8 != 0) + int((K if b_ld is None else b_ld) % 8 != 0 or k0 % 8 != 0)
            npieces += 1
            in_group += ln
            k0 += ln
            if in_group >= cap or npieces == max_seg:
                total, in_group, npieces = total + 1, 0, 0
    return total + (1 if npieces else 0) + copies


def blocked(gpu, rows, Ks, cols, cdt, ids=None, seed=0, lim=4):
    """A (len(rows) x len(Ks)) by (len(Ks) x len(cols)) grid of packed integer bf16 tiles through mb_matmul_blocked_subset
    (ids = None: every C block).  C blocks start as NaN (the call overwrites), those outside ids as -7 (must stay).
    Returns (per-C-block results, per-C-block references, launches, untouched-outside flags)."""
    lib, ctx = gpu
    m, k, n = len(rows), len(Ks), len(cols)
    rng = np.random.default_rng(seed)
    At = {(i, kk): ints(rng, (rows[i], Ks[kk]), lim) for i in range(m) for kk in range(k)}
    Bt = {(kk, j): ints(rng, (Ks[kk], cols[j]), lim) for kk in range(k) for j in range(n)}
    sa = {key: Stored(v, nat.MB_BF16) for key, v in At.items()}
    sb = {key: Stored(v, nat.MB_BF16) for key, v in Bt.items()}
    ids = list(range(m * n)) if ids is None else ids
    sc = {(i, j): Stored(np.full((rows[i], cols[j]), np.nan if i * n + j in ids else -7.0), cdt, fill=-7.0)
          for i in range(m) for j in range(n)}
    a_h = (nat.c_blk * (m * k))(*[sa[(i, kk)].block(gpu) for i in range(m) for kk in range(k)])
    b_h = (nat.c_blk * (k * n))(*[sb[(kk, j)].block(gpu) for kk in range(k) for j in range(n)])
    c_h = (nat.c_blk * (m * n))(*[sc[(i, j)].block(gpu) for i in range(m) for j in range(n)])
    l0 = launches(gpu)
    nat.check(lib.mb_matmul_blocked_subset(ctx, a_h, b_h, m, k, n, c_h, (C.c_int32 * len(ids))(*ids), len(ids)))
    sync(gpu)
    n_launch = launches(gpu) - l0
    for h in list(a_h) + list(b_h) + list(c_h):
        lib.mb_block_free(ctx, h)
    got, ref, outside = {}, {}, {}
    for (i, j), s in sc.items():
        got[(i, j)], outside[(i, j)] = s.read()
        if i * n + j not in ids:
            ref[(i, j)] = np.full((rows[i], cols[j]), -7.0)
        elif cdt == nat.MB_F32 or k <= 8:
            ref[(i, j)] = expected(np.hstack([At[(i, kk)] for kk in range(k)]), np.vstack([Bt[(kk, j)] for kk in range(k)]), cdt)
        else:   # more than 8 tiles: one product per launch, each accumulated into the bf16 block (one rounding each)
            acc = np.zeros((rows[i], cols[j]))
            for kk in range(k):
                acc = bf16_round(acc + At[(i, kk)] @ Bt[(kk, j)])
            ref[(i, j)] = acc
    return got, ref, n_launch, outside


def accuracy_errors(gpu, seed=7):
    """Max per-element error of an fp32 C at total K = 65536 against the fp64 product of the same bf16 inputs: through
    mb_matmul_blocked on (1,4,1) tiles of 256 x 16384 / 16384 x 256 and through one mb_block_gemm of 256 x 65536 x 256.
    U[0,1) data: |C - ref| / ref; U[-1,1) data: |C - ref| / (|A||B|)."""
    lib, ctx = gpu
    rng = np.random.default_rng(seed)
    m, K, n, k = 256, 65536, 256, 4
    out = {}
    for dist in ("u01", "u11"):
        A, B = rng.random((m, K)), rng.random((K, n))
        if dist == "u11":
            A, B = 2 * A - 1, 2 * B - 1
        A, B = to_bf16_values(A), to_bf16_values(B)
        ref = A @ B
        denom = ref if dist == "u01" else np.abs(A) @ np.abs(B)
        kt = K // k
        sa = [Stored(A[:, kk * kt:(kk + 1) * kt], nat.MB_BF16, pad=0) for kk in range(k)]
        sb = [Stored(B[kk * kt:(kk + 1) * kt], nat.MB_BF16, pad=0) for kk in range(k)]
        sc = Stored(np.zeros((m, n)), nat.MB_F32, pad=0)
        a_h = (nat.c_blk * k)(*[s.block(gpu) for s in sa])
        b_h = (nat.c_blk * k)(*[s.block(gpu) for s in sb])
        c_h = (nat.c_blk * 1)(sc.block(gpu))
        nat.check(lib.mb_matmul_blocked(ctx, a_h, b_h, 1, k, 1, c_h))
        sync(gpu)
        out[f"blocked_{dist}"] = float((np.abs(sc.values() - ref) / denom).max())
        whole_a, whole_b = Stored(A, nat.MB_BF16, pad=0), Stored(B, nat.MB_BF16, pad=0)
        ha, hb = whole_a.block(gpu), whole_b.block(gpu)
        nat.check(lib.mb_block_gemm(ctx, ha, hb, c_h[0], 0))
        sync(gpu)
        out[f"gemm_{dist}"] = float((np.abs(sc.values() - ref) / denom).max())
        for h in list(a_h) + list(b_h) + [c_h[0], ha, hb]:
            lib.mb_block_free(ctx, h)
    return out


# =========================================================================== 1. shapes x transposes x C layouts, exact
def test_bf16_round_matches_rne():
    rng = np.random.default_rng(1)
    x = np.concatenate([rng.integers(-70000, 70000, 2000).astype(np.float64), rng.standard_normal(2000) * 1e3,
                        [0.0, 257.0, 259.0, 261.0, 263.0, -257.0, 2.0 ** 20 + 2.0 ** 12]])
    assert np.array_equal(bf16_round(x), bf16_rne(x))


# (M, N, K): ragged tails against the 128 x 256 tile and the 64-wide k-slab, odd dimensions, and two multi-wave cases:
# 2181 x 1800 is 18 x 8 = 144 tiles (more than the 132 SMs: some CTAs run a second tile, crossing a 16-row band, with
# K = 136 = 3 slabs, so the smem ring's phase is out of step between a CTA's tiles); 4225 x 1793 is 34 x 8 = 272 tiles,
# more than two waves, ragged both ways.
SHAPES = [(1, 1, 8), (1, 264, 136), (64, 1, 72), (64, 40, 1000), (200, 264, 72), (200, 1800, 8), (2181, 40, 136),
          (2181, 1800, 136), (4225, 1793, 72), (37, 21, 13), (5, 3, 1), (333, 257, 130)]
# every shape with operands read in place ('aligned') and staged ('odd'), except 4225 x 1793 (host time): aligned only
LAYOUTS = [(s, lay) for s in SHAPES for lay in ("aligned", "odd") if not (lay == "odd" and s == (4225, 1793, 72))]


@pytest.mark.parametrize("shape,layout", LAYOUTS, ids=["x".join(map(str, s)) + "-" + lay for s, lay in LAYOUTS])
@pytest.mark.parametrize("ta", [0, 1])
@pytest.mark.parametrize("tb", [0, 1])
def test_block_gemm_exact(gpu, shape, ta, tb, layout):
    m, n, k = shape
    rng = np.random.default_rng(m * 7 + n * 5 + k * 3 + 2 * ta + tb)
    A, B = ints(rng, (m, k)), ints(rng, (k, n))
    C32, C16 = ints(rng, (m, n), 1000), ints(rng, (m, n), 64)          # accumulate onto nonzero integer C (exact in bf16)
    AB = A @ B
    for ct in (False, True):
        for cdt, C0 in ((nat.MB_F32, None), (nat.MB_BF16, None), (nat.MB_F32, C32), (nat.MB_BF16, C16)):
            got, clean, n_launch = block_gemm(gpu, A, B, ta, tb, cdt, C0=C0, ct=ct, layout=layout)
            want = AB + (0.0 if C0 is None else C0)
            want = want if cdt == nat.MB_F32 else bf16_round(want)
            case = (shape, ta, tb, layout, ct, cdt, C0 is not None)
            assert np.array_equal(got, want), (case, np.argwhere(got != want)[:5], np.abs(got - want).max())
            assert clean, ("C's parent changed outside C",) + case
            if layout == "aligned":
                assert n_launch == 1, case                                  # read in place: one launch, no copy


# ==================================================================== 2. segment path of mb_matmul_blocked_subset, exact
# (rows, K per tile, cols).  Multiples of 8 are read in place; 130, 13 and 37-row tiles (ld 37) are staged.
GRIDS = [([200], [72, 136], [264]),
         ([200, 64], [72, 136, 8, 72], [264, 40]),
         ([64], [72, 136, 8, 72, 136, 8, 72, 136], [264]),
         ([37, 64], [130, 72, 13, 8], [21, 264]),
         ([136], [72] * 9, [264])]                        # k = 9: more than 8 segments, one launch per product


@pytest.mark.parametrize("grid", range(len(GRIDS)))
@pytest.mark.parametrize("cdt", [nat.MB_F32, nat.MB_BF16], ids=["f32", "bf16"])
def test_blocked_segments_exact(gpu, grid, cdt):
    rows, Ks, cols = GRIDS[grid]
    got, ref, n_launch, clean = blocked(gpu, rows, Ks, cols, cdt, seed=grid)
    for key in got:
        assert np.array_equal(got[key], ref[key]), (grid, key, np.abs(got[key] - ref[key]).max())
        assert clean[key], (grid, key)
    if len(Ks) <= 8:
        want = sum(chain_launches(Ks, KCHAIN_DEFAULT, r, cdt == nat.MB_F32) for r in rows for _ in cols)
    else:
        want = len(rows) * len(cols) * len(Ks)
    assert n_launch == want, (grid, n_launch, want)
    if grid in (0, 1, 2):
        assert n_launch == len(rows) * len(cols)                    # one launch per C block on the segment path


@pytest.mark.parametrize("cdt", [nat.MB_F32, nat.MB_BF16], ids=["f32", "bf16"])
def test_blocked_subset_leaves_other_blocks(gpu, cdt):
    got, ref, n_launch, clean = blocked(gpu, [64, 200, 37], [72, 130], [40, 264], cdt, ids=[5, 0, 3], seed=11)
    for key in got:
        assert np.array_equal(got[key], ref[key]), key
        assert clean[key], key


# ===================================================================================== 3. K-chain split, exact
# (rows, K per tile, cols, launches with the default cap of 8192)
CHAINS = [([136], [4000] * 3, [264], 2),            # 4000 + 4000 + 192 | 3808: the cut at k0 = 192 inside the last tile
          ([64], [1104] * 8, [40], 2)]              # 7 x 1104 + 464 (8 segments) | 640


@pytest.mark.parametrize("chain", range(len(CHAINS)))
def test_kchain_split_exact(gpu, chain):
    rows, Ks, cols, want = CHAINS[chain]
    got, ref, n_launch, clean = blocked(gpu, rows, Ks, cols, nat.MB_F32, seed=20 + chain)
    assert np.array_equal(got[(0, 0)], ref[(0, 0)])
    assert n_launch == want == chain_launches(Ks, KCHAIN_DEFAULT, rows[0])
    # the same product as ONE block GEMM is split by the same cap (first launch overwrites, the next add)
    rng = np.random.default_rng(30 + chain)
    A, B = ints(rng, (rows[0], sum(Ks))), ints(rng, (sum(Ks), cols[0]))
    for C0 in (None, ints(rng, (rows[0], cols[0]), 1000)):
        c, clean, n1 = block_gemm(gpu, A, B, 0, 0, nat.MB_F32, C0=C0)
        assert np.array_equal(c, expected(A, B, nat.MB_F32, C0)) and clean
        assert n1 == -(-sum(Ks) // KCHAIN_DEFAULT)
    c, clean, n1 = block_gemm(gpu, A, B, 1, 1, nat.MB_BF16)          # bf16 C: one launch, one rounding
    assert np.array_equal(c, expected(A, B, nat.MB_BF16)) and clean and n1 == 1


CAPS = [96, 1000, 100, 0]


@pytest.fixture(scope="module")
def kchain_workers():
    """The cap is read once per process: each other value runs in a fresh one (tests/bf16_kchain_worker.py), all four
    started together on first use."""
    procs = {cap: subprocess.Popen([sys.executable, str(ROOT / "tests" / "bf16_kchain_worker.py")], stdout=subprocess.PIPE,
                                   stderr=subprocess.STDOUT, text=True, cwd=str(ROOT),
                                   env=dict(os.environ, MARLIN_B200_BF16_KCHAIN=str(cap)))
             for cap in CAPS}
    yield procs
    for p in procs.values():
        if p.poll() is None:
            p.kill()
        p.wait()


@pytest.mark.parametrize("cap", CAPS)
def test_kchain_caps_in_subprocess(kchain_workers, cap):
    p = kchain_workers[cap]
    stdout, _ = p.communicate(timeout=600)
    assert p.returncode == 0, stdout[-4000:]
    res = json.loads(stdout.strip().splitlines()[-1])
    assert res["cap"] == cap and res["cases"] >= 4
    if cap == 0:
        # reported, not asserted: one 65536-long chain on U[0,1) data is what the cap exists to avoid (on an H100
        # 80GB HBM3 it measured 3.5e-4, above the 1e-4 tolerance; 3.1e-5 with the default cap)
        print(f"K = 65536, unlimited chains: {res['errors']}")
        assert len(res["errors"]) == 4 and all(np.isfinite(list(res["errors"].values())))


# =================================================================================== 4. views in poisoned parents
@pytest.mark.parametrize("aligned", [True, False], ids=["aligned", "unaligned"])
@pytest.mark.parametrize("ta", [0, 1])
@pytest.mark.parametrize("tb", [0, 1])
def test_views_in_poisoned_parents(gpu, aligned, ta, tb):
    """A and B as views inside NaN-filled bf16 parents (aligned offsets: read in place; unaligned: staged), C as a view
    inside a sentinel-filled fp32 or bf16 parent.  Random data: bit-identical to the same call on packed copies with ld
    a multiple of 8, and nothing outside C changes."""
    lib, ctx = gpu
    m, n, k = 150, 300, 200
    rng = np.random.default_rng(40 + 2 * ta + tb + 4 * aligned)
    A, B = to_bf16_values(rng.random((m, k)) - 0.5), to_bf16_values(rng.random((k, n)) - 0.5)
    r0, c0 = (8, 3) if aligned else (3, 5)

    def view(x, trans):
        s = x.T if trans else x
        pr = s.shape[0] + r0 + (5 if aligned else 4)
        pr = -(-pr // 8) * 8 if aligned else pr | 1           # parent ld: a multiple of 8, or odd
        parent = np.full((pr, s.shape[1] + c0 + 7), np.nan)
        parent[r0:r0 + s.shape[0], c0:c0 + s.shape[1]] = s
        p = Stored(parent, nat.MB_BF16)
        h = nat.c_blk()
        nat.check(lib.mb_block_slice(ctx, p.block(gpu), r0, r0 + s.shape[0], c0, c0 + s.shape[1], C.byref(h)))
        if trans:
            v = nat.c_blk()
            nat.check(lib.mb_block_view_t(ctx, h, C.byref(v)))
            h = v
        return p, h

    pa, ha = view(A, ta)
    pb, hb = view(B, tb)
    for cdt, sentinel in ((nat.MB_F32, 12345.5), (nat.MB_BF16, -3.0)):
        for acc in (0, 1):
            want, _, _ = block_gemm(gpu, A, B, ta, tb, cdt, C0=np.ones((m, n)) if acc else None)
            cpar = np.full((m + 11, n + 6), sentinel)
            cpar[4:4 + m, 2:2 + n] = 1.0 if acc else np.nan
            pc = Stored(cpar, cdt)
            hc = nat.c_blk()
            nat.check(lib.mb_block_slice(ctx, pc.block(gpu), 4, 4 + m, 2, 2 + n, C.byref(hc)))
            nat.check(lib.mb_block_gemm(ctx, ha, hb, hc, acc))
            sync(gpu)
            got = pc.values()
            assert np.array_equal(got[4:4 + m, 2:2 + n], want), (cdt, acc)
            outside = np.ones(cpar.shape, dtype=bool)
            outside[4:4 + m, 2:2 + n] = False
            assert np.all(got[outside] == sentinel) and pc.untouched_outside(), (cdt, acc)
    assert pa.untouched_outside() and pb.untouched_outside()


# ====================================================================== 5. accuracy at config-5 chain length (default cap)
def test_accuracy_at_config5_chain_length(gpu):
    errs = accuracy_errors(gpu)
    print(f"K = 65536, chains capped at {KCHAIN_DEFAULT}: {errs}")
    for key, err in errs.items():
        assert err <= 1e-4, (key, err)


# ============================================================================================== 6. small cases
@pytest.mark.parametrize("cdt", [nat.MB_F32, nat.MB_BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("ct", [False, True])
def test_k_zero(gpu, cdt, ct):
    """K = 0: C := 0 (from NaN), or C unchanged under accumulate, as the fp64 path does."""
    A, B = np.zeros((40, 0)), np.zeros((0, 264))
    got, clean, _ = block_gemm(gpu, A, B, 0, 0, cdt, ct=ct)
    assert np.array_equal(got, np.zeros((40, 264))) and not np.signbit(got).any() and clean
    C0 = ints(np.random.default_rng(2), (40, 264), 64)
    got, clean, n_launch = block_gemm(gpu, A, B, 1, 0, cdt, C0=C0, ct=ct)
    assert np.array_equal(got, C0) and clean and n_launch == 0


def test_k_zero_blocked(gpu):
    got, ref, _, clean = blocked(gpu, [37], [0, 0], [21], nat.MB_F32)
    assert np.array_equal(got[(0, 0)], np.zeros((37, 21))) and clean[(0, 0)]


@pytest.mark.parametrize("mn", [(0, 40), (40, 0), (0, 0)])
def test_empty_result_is_a_no_op(gpu, mn):
    m, n = mn
    rng = np.random.default_rng(3)
    got, clean, n_launch = block_gemm(gpu, ints(rng, (m, 24)), ints(rng, (24, n)), 0, 0, nat.MB_F32)
    assert got.shape == (m, n) and clean and n_launch == 0


def test_fp64_times_bf16_is_unsupported(gpu):
    lib, ctx = gpu
    a = Stored(np.ones((16, 16)), nat.MB_F64)
    b = Stored(np.ones((16, 16)), nat.MB_BF16)
    c = Stored(np.zeros((16, 16)), nat.MB_F32)
    assert lib.mb_block_gemm(ctx, a.block(gpu), b.block(gpu), c.block(gpu), 0) == nat.MB_ERR_UNSUPPORTED
    assert lib.mb_block_gemm(ctx, b.block(gpu), a.block(gpu), c.block(gpu), 0) == nat.MB_ERR_UNSUPPORTED


# ============================================================================================ 7. Python level
def test_random_block_matrix_3x3_bf16():
    """1000 x 1000 on a 3 x 3 grid: 334- and 332-row blocks, packed with ld = rows, so most operands are staged."""
    import marlin_b200 as mb
    mb.Runtime.get()
    A = mb.MTUtils.randomBlockMatrix(None, 1000, 1000, 3, 3, seed=31, dtype=nat.MB_BF16)
    B = mb.MTUtils.randomBlockMatrix(None, 1000, 1000, 3, 3, seed=32, dtype=nat.MB_BF16)
    got = A.multiply(B).toBreeze()
    ref = A.toBreeze() @ B.toBreeze()
    assert (np.abs(got - ref) / ref).max() <= 1e-4

"""Every fp64 DMMA path on exact integer data, compared with `==` against the host product (tests/exact_gemm.py).

Integer operands whose worst case |alpha| K max|a| max|b| + |beta| max|c| lies in [2^52, 2^53] make every summation
order, k split and DMMA shape give the same fp64 number, and use the whole significand: a dropped term, a narrowed
accumulator, a tile stored to the wrong place or never stored (outputs start as NaN) all show as a mismatch, whatever
order a kernel sums in.  This net, not bit-equality with the m8n8k4 instances, is what a mainloop change that reorders k
within an instruction or changes which CTA loads a slab has to pass.

Every case also checks which kernel ran, by name through torch.profiler, and where a launch count is the claim (the
grouped launch against its per-product fallback, the host pipelines' K split and column chunks, the row-shard chunks)
through mb_launch_count.
"""
import ctypes as C
import functools
import itertools
import re

import numpy as np
import pytest

from marlin_b200 import _native as nat
from tests import exact_gemm as xg
from tests.harness import gpu  # noqa: F401  (a fixture)
from tests.test_gpu_bf16_exact import Stored

pytestmark = pytest.mark.gpu
F64 = nat.MB_F64
DMMA = "gemm_f64_dmma16x8_kernel"
GROUPED = "gemm_f64_dmma16x8_grouped_kernel"
GENERIC = "gemm_f64_generic_kernel"
FORMS = [(0, 0), (1, 0), (0, 1), (1, 1)]
FORM_IDS = ["NN", "TN", "NT", "TT"]


# ------------------------------------------------------------------------------------------------------------ helpers
def even(x):
    return max(2, (x + 1) & ~1)


def _norm(name):
    """A kernel name with its template arguments spelled true / false and no spaces."""
    return re.sub(r"\(bool\)1", "true", re.sub(r"\(bool\)0", "false", name)).replace(" ", "")


def form(kernel, ta, tb):
    return f"{kernel}<{'true' if ta else 'false'},{'true' if tb else 'false'}>"


def profiled(gpu, fn, reference=False):
    """fn() with the m8n8k4 reference kernels on or off: (its result, the library's kernel names, library launches).

    The trace can miss kernels launched right after it starts: a multiply that launched its one grouped kernel at once
    has come back with an empty trace, and one that launched a GEMM and then a transpose with the transpose alone.  So a
    torch kernel runs and completes inside the trace before fn starts, and a trace without any library kernel is a
    capture the profiler missed (every fn here launches at least one): fn runs again, at most twice more.  fn builds its
    own outputs, so its result does not depend on the attempt.  mb_launch_count does not depend on the profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    lib, ctx = gpu
    nat.check(lib.mb_set_dmma_reference(ctx, int(reference)))
    try:
        for _ in range(3):
            torch.cuda.synchronize()
            l0 = lib.mb_launch_count(ctx)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                torch.ones(1, device="cuda").add_(1.0)
                torch.cuda.synchronize()
                out = fn()
                torch.cuda.synchronize()
            launches = lib.mb_launch_count(ctx) - l0
            names = {_norm(e.name) for e in prof.events()
                     if e.device_type.name == "CUDA" and re.search(r"(^|\W)mb::", e.name)}
            if names:
                break
    finally:
        nat.check(lib.mb_set_dmma_reference(ctx, 0))
    return out, names, launches


def only(names, *kernels):
    """Every library kernel that ran is one of `kernels`, and each of them ran."""
    assert names and all(any(k in n for k in kernels) for n in names), sorted(names)
    assert all(any(k in n for n in names) for k in kernels), (kernels, sorted(names))


@functools.lru_cache(maxsize=None)
def case(m, k, n, alpha=1.0, beta=0.0, seed=0):
    """Operands and exact reference of one shape, shared between the forms and layouts that use it."""
    rng = np.random.default_rng([m, k, n, seed, int(alpha * 16) + 100, int(beta) + 10])
    A, B, C0 = xg.operands(rng, m, k, n, alpha, beta)
    return A, B, C0, xg.reference(A, B, alpha, beta, C0)


def ptr(s):
    return C.c_void_p(s.t.data_ptr() + 8 * s.offset)


def dgemm(gpu, ta, tb, A, B, alpha=1.0, beta=0.0, C0=None, lay_a=(None, 0), lay_b=(None, 0), lay_c=(None, 0)):
    """mb_dgemm_device on A, B given logically and stored as op() needs them, each in a NaN-filled flat tensor at
    (ld, offset) (ld None: rows rounded up to even); C starts as NaN unless beta != 0.  Returns (C, padding untouched)."""
    lib, ctx = gpu
    m, k = A.shape
    n = B.shape[1]
    sa, sb = (A.T if ta else A), (B.T if tb else B)
    Sa = Stored(sa, F64, ld=lay_a[0] or even(sa.shape[0]), offset=lay_a[1])
    Sb = Stored(sb, F64, ld=lay_b[0] or even(sb.shape[0]), offset=lay_b[1])
    Sc = Stored(C0 if beta != 0.0 else np.full((m, n), np.nan), F64, ld=lay_c[0] or even(m), offset=lay_c[1])
    nat.check(lib.mb_dgemm_device(ctx, b"T" if ta else b"N", b"T" if tb else b"N", m, n, k, alpha, ptr(Sa), Sa.ld,
                                  ptr(Sb), Sb.ld, beta, ptr(Sc), Sc.ld))
    nat.check(lib.mb_synchronize(ctx))              # the library's stream, not torch's, runs the kernel
    got, clean = Sc.read()
    return got, clean and Sa.untouched_outside() and Sb.untouched_outside()


def check_all(results):
    for what, got, want, clean in results:
        xg.assert_exact(got, want, what)
        assert clean, f"{what}: memory outside the matrices changed"


# ============================================================================ a. mb_dgemm_device: tiles, ring, waves
EDGE_MN = [1, 2, 127, 128, 129, 255]
EDGE_K = [1, 15, 16, 17, 95, 96, 97, 4099]          # BK = 16; 96 = the 6-stage ring, where the phase first flips


@pytest.mark.parametrize("ta,tb", FORMS, ids=FORM_IDS)
def test_dgemm_tile_and_ring_edges(gpu, ta, tb):
    shapes = [(m, k, n) for m in EDGE_MN for n in EDGE_MN for k in EDGE_K]

    def fn():
        out = []
        for m, k, n in shapes:
            A, B, _, want = case(m, k, n)
            got, clean = dgemm(gpu, ta, tb, A, B)
            out.append(((m, k, n), got, want, clean))
        return out

    res, names, launches = profiled(gpu, fn)
    only(names, form(DMMA, ta, tb))
    assert launches == len(shapes)
    check_all(res)


# (M, K, N): tiles on 132 SMs.  1536 x 1408 = 12 x 11 = 132 (exactly one wave); 1537 x 1408 = 13 x 11 = 143;
# 2049 x 2048 = 17 x 16 = 272 tiles, more than two waves, and tiles_m = 17 ends on a one-row band after a full band of 16;
# 4000 x 1100 = 32 x 9 = 288.  K = 97, 200 and 1000 are 7, 13 and 63 slabs: not whole ring cycles, so a persistent CTA
# starts its next tile mid-cycle.
WAVES = [(1536, 97, 1408), (1537, 200, 1408), (2049, 1000, 2048), (4000, 97, 1100)]


@pytest.mark.parametrize("ta,tb", FORMS, ids=FORM_IDS)
def test_dgemm_wave_edges(gpu, ta, tb):
    def fn():
        out = []
        for m, k, n in WAVES:
            A, B, _, want = case(m, k, n)
            got, clean = dgemm(gpu, ta, tb, A, B)
            out.append(((m, k, n), got, want, clean))
        return out

    res, names, launches = profiled(gpu, fn)
    only(names, form(DMMA, ta, tb))
    assert launches == len(WAVES)
    check_all(res)


@pytest.mark.parametrize("ta,tb", [(0, 0), (1, 1)], ids=["NN", "TT"])
def test_dgemm_4096_cubed(gpu, ta, tb):
    A, B, _, want = case(4096, 4096, 4096)
    (got, clean), names, launches = profiled(gpu, lambda: dgemm(gpu, ta, tb, A, B))
    only(names, form(DMMA, ta, tb))
    assert launches == 1 and clean
    xg.assert_exact(got, want, f"4096^3 {ta}{tb}")


ALPHA_BETA = list(itertools.product([1.0, -3.0, 2.0 ** -4], [0.0, 1.0, -2.0]))
# C layouts: 16-byte aligned with even ldc (16-byte stores), an odd element offset, an odd ldc (scalar stores; at
# beta != 0 add versus add2).  Every ldc leaves padding between columns, which must come back untouched.
C_LAYOUTS = {"aligned": lambda m: (even(m) + 2, 0), "odd_offset": lambda m: (even(m) + 2, 1),
             "odd_ldc": lambda m: (even(m) + 3, 0)}


@pytest.mark.parametrize("ta,tb", FORMS, ids=FORM_IDS)
def test_dgemm_epilogue(gpu, ta, tb):
    m, k, n = 300, 97, 259

    def fn():
        out = []
        for (alpha, beta), (lay, ldc) in itertools.product(ALPHA_BETA, C_LAYOUTS.items()):
            A, B, C0, want = case(m, k, n, alpha, beta)
            got, clean = dgemm(gpu, ta, tb, A, B, alpha, beta, C0, lay_c=ldc(m))
            out.append(((alpha, beta, lay), got, want, clean))
        return out

    res, names, launches = profiled(gpu, fn)
    only(names, form(DMMA, ta, tb))
    assert launches == len(ALPHA_BETA) * len(C_LAYOUTS)
    check_all(res)


# operand layouts around TMA eligibility: 16-byte aligned with even ld (DMMA), one element off (generic), odd ld (generic)
OPERAND_LAYOUTS = [("aligned", lambda r: (even(r) + 2, 2), DMMA), ("offset1", lambda r: (even(r), 1), GENERIC),
                   ("odd_ld", lambda r: (even(r) + 1, 0), GENERIC)]


@pytest.mark.parametrize("ta,tb", FORMS, ids=FORM_IDS)
@pytest.mark.parametrize("which", ["A", "B"])
@pytest.mark.parametrize("layout", range(len(OPERAND_LAYOUTS)), ids=[x[0] for x in OPERAND_LAYOUTS])
def test_dgemm_tma_eligibility(gpu, ta, tb, which, layout):
    m, k, n = 200, 97, 150
    A, B, _, want = case(m, k, n)
    _, lay, kernel = OPERAND_LAYOUTS[layout]
    rows = (k if ta else m) if which == "A" else (n if tb else k)
    kw = {"lay_a" if which == "A" else "lay_b": lay(rows)}
    (got, clean), names, launches = profiled(gpu, lambda: dgemm(gpu, ta, tb, A, B, -3.0, 0.0, None, **kw))
    only(names, form(kernel, ta, tb))
    assert launches == 1 and clean
    xg.assert_exact(got, -3.0 * want, f"{which} {OPERAND_LAYOUTS[layout][0]}")


@pytest.mark.parametrize("ta,tb", FORMS, ids=FORM_IDS)
def test_dgemm_reference_instances(gpu, ta, tb):
    """The m8n8k4 instances that test_gpu_dmma_reference.py compares against are themselves exact."""
    shapes = [(129, 97, 255), (2049, 200, 2048)] if (ta, tb) == (0, 0) else [(129, 97, 255)]

    def fn():
        return [((m, k, n), *dgemm(gpu, ta, tb, case(m, k, n)[0], case(m, k, n)[1])) for m, k, n in shapes]

    res, names, launches = profiled(gpu, fn, reference=True)
    only(names, form("gemm_f64_dmma_kernel", ta, tb))
    assert launches == len(shapes)
    for (shape, got, clean) in res:
        xg.assert_exact(got, case(*shape)[3], f"m8n8k4 {shape}")
        assert clean


# ================================================================================== b. mb_block_gemm on views
def view_in_parent(gpu, x, trans, r0=2, c0=3):
    """x as a slice at (r0, c0) of a NaN-filled column-major parent (even ld, so the slice stays 16-byte aligned), or
    as the transpose view of such a slice of x^T.  Returns (parent, block handle)."""
    lib, ctx = gpu
    s = x.T if trans else x
    parent = np.full((even(s.shape[0] + r0 + 3), s.shape[1] + c0 + 2), np.nan)
    parent[r0:r0 + s.shape[0], c0:c0 + s.shape[1]] = s
    p = Stored(parent, F64)
    h = nat.c_blk()
    nat.check(lib.mb_block_slice(ctx, p.block(gpu), r0, r0 + s.shape[0], c0, c0 + s.shape[1], C.byref(h)))
    if trans:
        v = nat.c_blk()
        nat.check(lib.mb_block_view_t(ctx, h, C.byref(v)))
        h = v
    return p, h


@pytest.mark.parametrize("ta,tb", FORMS, ids=FORM_IDS)
@pytest.mark.parametrize("ct", [False, True], ids=["C", "Crow"])
def test_block_gemm_views(gpu, ta, tb, ct):
    """Operands and C as slices of NaN-filled parents; transposed-view operands; a row-major (transposed-view) C, run as
    C^T = B^T A^T; overwrite and accumulate.  Nothing outside C may change."""
    lib, ctx = gpu
    m, k, n = 300, 1000, 260
    out_form = (1 - tb, 1 - ta) if ct else (ta, tb)

    def fn():
        out = []
        for acc in (0, 1):
            A, B, C0, want = case(m, k, n, 1.0, float(acc), seed=1)
            pa, ha = view_in_parent(gpu, A, ta)
            pb, hb = view_in_parent(gpu, B, tb, 4, 1)
            pc, hc = view_in_parent(gpu, C0 if acc else np.full((m, n), np.nan), ct, 6, 2)
            nat.check(lib.mb_block_gemm(ctx, ha, hb, hc, acc))
            nat.check(lib.mb_synchronize(ctx))
            cs = (n, m) if ct else (m, n)
            par = pc.values()
            got = par[6:6 + cs[0], 2:2 + cs[1]]
            rest = par.copy()
            rest[6:6 + cs[0], 2:2 + cs[1]] = np.nan
            clean = bool(np.all(np.isnan(rest))) and pc.untouched_outside() and pa.untouched_outside() and pb.untouched_outside()
            out.append((("acc", acc), got.T if ct else got, want, clean))
        return out

    res, names, launches = profiled(gpu, fn)
    only(names, form(DMMA, *out_form))
    assert launches == 2
    check_all(res)


# ========================================================================================= c. mb_dgemm_host
HOST_SHAPES = [(33, 41, 29), (128, 97, 129), (255, 1000, 2), (1, 17, 300), (257, 4099, 131)]


@pytest.mark.parametrize("ta,tb", FORMS, ids=FORM_IDS)
def test_dgemm_host(gpu, ta, tb):
    """Host arrays with non-zero offsets, leading dimensions larger than needed and beta != 0 (the netlib signature);
    the padding between columns of C comes back untouched."""
    lib, ctx = gpu

    def fn():
        out = []
        for idx, (m, k, n) in enumerate(HOST_SHAPES):
            alpha, beta = ALPHA_BETA[(3 * idx + 1) % len(ALPHA_BETA)]
            beta = beta or 1.0
            A, B, C0, want = case(m, k, n, alpha, beta, seed=2)
            sa, sb = (A.T if ta else A), (B.T if tb else B)
            offs, lds = (7, 3, 5), (sa.shape[0] + 3, sb.shape[0] + 4, m + 5)
            arrs = []
            for x, off, ld in zip((sa, sb, C0), offs, lds):
                flat = np.full(off + ld * x.shape[1] + 3, -7.25)
                flat[off:off + ld * x.shape[1]].reshape(x.shape[1], ld)[:, :x.shape[0]] = x.T
                arrs.append(flat)
            c_before = arrs[2].copy()
            nat.check(lib.mb_dgemm_host(ctx, b"T" if ta else b"N", b"T" if tb else b"N", m, n, k, alpha,
                                        arrs[0].ctypes.data_as(C.c_void_p), offs[0], lds[0],
                                        arrs[1].ctypes.data_as(C.c_void_p), offs[1], lds[1], beta,
                                        arrs[2].ctypes.data_as(C.c_void_p), offs[2], lds[2]))
            win = arrs[2][offs[2]:offs[2] + lds[2] * n].reshape(n, lds[2])
            pad = np.ones(len(c_before), bool)
            pad[offs[2]:offs[2] + lds[2] * n].reshape(n, lds[2])[:, :m] = False
            out.append(((m, k, n, alpha, beta), win[:, :m].T.copy(), want, bool(np.array_equal(arrs[2][pad], c_before[pad]))))
        return out

    res, names, launches = profiled(gpu, fn)
    only(names, form(DMMA, ta, tb))
    assert launches == len(HOST_SHAPES)
    check_all(res)


# ========================================================================= d. grouped blocked multiply (one launch)
def blocked(gpu, rows, ks, cols, ids=None, odd_tile=None, seed=0):
    """An (len(rows) x len(ks)) by (len(ks) x len(cols)) grid of integer fp64 tiles through mb_matmul_blocked_subset
    (ids None: every C block), profiled.  A tiles have ld = rows rounded up to even; B tiles ld = k rounded up to even,
    so a ragged K segment has NaN rows under it that the kernel must never read; odd_tile = (i, kk): that A tile with
    an odd ld instead.  C blocks in ids start as NaN, the others hold the sentinel -7 and must keep it.  Returns ({C
    block: (got, want, untouched outside)}, kernel names, launches)."""
    lib, ctx = gpu
    m, k, n = len(rows), len(ks), len(cols)
    rng = np.random.default_rng(seed)
    A, B, _ = xg.operands(rng, sum(rows), sum(ks), sum(cols))
    ref = xg.reference(A, B)
    r0, k0, c0 = np.cumsum([0] + rows), np.cumsum([0] + ks), np.cumsum([0] + cols)
    ids = list(range(m * n)) if ids is None else ids

    def fn():
        sa = {(i, kk): Stored(A[r0[i]:r0[i + 1], k0[kk]:k0[kk + 1]], F64,
                              ld=rows[i] + (1 if rows[i] % 2 == 0 else 0) if (i, kk) == odd_tile else even(rows[i]))
              for i in range(m) for kk in range(k)}
        sb = {(kk, j): Stored(B[k0[kk]:k0[kk + 1], c0[j]:c0[j + 1]], F64, ld=even(ks[kk])) for kk in range(k) for j in range(n)}
        sc = {(i, j): Stored(np.full((rows[i], cols[j]), np.nan if i * n + j in ids else -7.0), F64, ld=even(rows[i]),
                             fill=np.nan if i * n + j in ids else -7.0) for i in range(m) for j in range(n)}
        a_h = (nat.c_blk * (m * k))(*[sa[(i, kk)].block(gpu) for i in range(m) for kk in range(k)])
        b_h = (nat.c_blk * (k * n))(*[sb[(kk, j)].block(gpu) for kk in range(k) for j in range(n)])
        c_h = (nat.c_blk * (m * n))(*[sc[(i, j)].block(gpu) for i in range(m) for j in range(n)])
        nat.check(lib.mb_matmul_blocked_subset(ctx, a_h, b_h, m, k, n, c_h, (C.c_int32 * len(ids))(*ids), len(ids)))
        nat.check(lib.mb_synchronize(ctx))
        for h in list(a_h) + list(b_h) + list(c_h):
            lib.mb_block_free(ctx, h)
        out = {}
        for (i, j), s in sc.items():
            got, clean = s.read()
            want = ref[r0[i]:r0[i + 1], c0[j]:c0[j + 1]] if i * n + j in ids else np.full((rows[i], cols[j]), -7.0)
            out[(i, j)] = (got, want, clean and all(x.untouched_outside() for x in list(sa.values()) + list(sb.values())))
        return out

    return profiled(gpu, fn)


def check_blocks(res, what):
    for key, (got, want, clean) in sorted(res.items()):
        xg.assert_exact(got, want, f"{what} C{key}")
        assert clean, (what, key)


def test_grouped_ragged_k_segments(gpu):
    """K segments of 1, 15, 17 and 1000 in one entry: every segment's zero-filled tail adds exact zeros (the NaN rows
    under each B tile are never read)."""
    res, names, launches = blocked(gpu, [300], [1, 15, 17, 1000], [260])
    only(names, GROUPED)
    assert launches == 1
    check_blocks(res, "ragged K")


def test_grouped_entries_of_different_sizes(gpu):
    """Entries of 144, 16, 18 and 2 tiles (180 in all): persistent CTAs cross from one entry into the next."""
    res, names, launches = blocked(gpu, [2000, 130], [64, 33], [1100, 40], seed=1)
    only(names, GROUPED)
    assert launches == 1
    check_blocks(res, "mixed entries")


def test_grouped_more_than_two_waves(gpu):
    """Four entries of 9 x 9 tiles: 324 tiles in one launch, 2.45 waves on 132 SMs."""
    res, names, launches = blocked(gpu, [1100, 1100], [100, 50, 6], [1100, 1100], seed=2)
    only(names, GROUPED)
    assert launches == 1
    check_blocks(res, "three waves")


# (name, rows, ks, cols): each limit of the grouped launch exactly at (one launch) and one past (the fallback: one
# launch per product, m * n * k).  K segments <= 16; entries (C blocks) <= 64; operand tiles per side <= 32.
LIMITS = [("k16", [40], [20] * 16, [36], True), ("k17", [40], [20] * 17, [36], False),
          ("c64", [16] * 8, [20], [16] * 8, True), ("c65", [16] * 5, [20], [16] * 13, False),
          ("a32", [16, 16], [8] * 16, [24], True), ("a33", [16, 16, 16], [8] * 11, [24], False),
          ("b32", [24], [8] * 16, [16, 16], True), ("b33", [24], [8] * 11, [16, 16, 16], False)]


@pytest.mark.parametrize("limit", range(len(LIMITS)), ids=[x[0] for x in LIMITS])
def test_grouped_limits(gpu, limit):
    name, rows, ks, cols, grouped = LIMITS[limit]
    res, names, launches = blocked(gpu, rows, ks, cols, seed=3 + limit)
    if grouped:
        only(names, GROUPED)
        assert launches == 1, name
    else:
        only(names, form(DMMA, 0, 0))
        assert launches == len(rows) * len(ks) * len(cols), name
    check_blocks(res, name)


def test_grouped_odd_ld_tile_falls_back(gpu):
    """One A tile with an odd ld cannot be read by TMA: the whole call runs per product (that product on the CUDA
    cores), still exact."""
    res, names, launches = blocked(gpu, [300, 64], [40, 40], [50], odd_tile=(1, 1), seed=11)
    only(names, form(DMMA, 0, 0), form(GENERIC, 0, 0))
    assert launches == 4
    check_blocks(res, "odd ld")


def test_grouped_subset(gpu):
    """Only the listed C blocks are computed; every other block keeps its sentinel."""
    res, names, launches = blocked(gpu, [64, 200, 37], [72, 130], [40, 264], ids=[5, 0, 3], seed=12)
    only(names, GROUPED)
    assert launches == 1
    check_blocks(res, "subset")


# ============================================================================================= e. host pipelines
def blocked_host_launches(rows, ks, cols):
    """DMMA launches of mb_matmul_blocked_host: the first product split in 4 along K when k >= 1024 (unless it is also the
    last), the first and the last product in 4 column chunks when their C block has >= 1024 columns, 1 otherwise."""
    m, k, n = len(rows), len(ks), len(cols)
    total = 0
    for i, j, kk in itertools.product(range(m), range(n), range(k)):
        first, last = (i, j, kk) == (0, 0, 0), (i, j, kk) == (m - 1, n - 1, k - 1)
        if first and not last and ks[kk] >= 1024:
            total += 4
        else:
            total += 4 if (first or last) and cols[j] >= 1024 else 1
    return total


def run_blocked_host(gpu, rows, ks, cols, seed):
    lib, ctx = gpu
    m, k, n = len(rows), len(ks), len(cols)
    rng = np.random.default_rng(seed)
    A, B, _ = xg.operands(rng, sum(rows), sum(ks), sum(cols))
    ref = xg.reference(A, B)
    r0, k0, c0 = np.cumsum([0] + rows), np.cumsum([0] + ks), np.cumsum([0] + cols)
    a = [np.asfortranarray(A[r0[i]:r0[i + 1], k0[kk]:k0[kk + 1]]) for i in range(m) for kk in range(k)]
    b = [np.asfortranarray(B[k0[kk]:k0[kk + 1], c0[j]:c0[j + 1]]) for kk in range(k) for j in range(n)]

    def fn():
        c = [np.full((rows[i], cols[j]), np.nan, order="F") for i in range(m) for j in range(n)]
        nat.check(lib.mb_matmul_blocked_host(ctx, (C.c_void_p * (m * k))(*[x.ctypes.data for x in a]),
                                             (C.c_void_p * (k * n))(*[x.ctypes.data for x in b]), m, k, n,
                                             (C.c_int32 * m)(*rows), (C.c_int32 * k)(*ks), (C.c_int32 * n)(*cols),
                                             (C.c_void_p * (m * n))(*[x.ctypes.data for x in c])))
        return c

    c, names, launches = profiled(gpu, fn)
    only(names, form(DMMA, 0, 0))
    assert launches == blocked_host_launches(rows, ks, cols), (rows, ks, cols, launches)
    for i, j in itertools.product(range(m), range(n)):
        xg.assert_exact(c[i * n + j], ref[r0[i]:r0[i + 1], c0[j]:c0[j + 1]], f"{rows}x{ks}x{cols} C({i},{j})")


def test_matmul_blocked_host(gpu):
    """On a fresh context: a small call, the same call again (workspace reused), then larger ones (workspace regrown).
    K split of the first product at k = 1030 and 4097 (cut points rounded down to multiples of 16, the last chunk ending
    at k); column-chunked upload (first product) and download (last product) at >= 1024 columns; a 1 x 1 x 1 grid whose
    only product is first and last, so it skips the K split and is column-chunked both ways."""
    lib = gpu[0]
    ctx = nat.c_ctx()
    nat.check(lib.mb_init(0, C.byref(ctx)))
    try:
        g = (lib, ctx)
        small = ([130, 40], [300, 20], [1200, 50])            # first product column-chunked (upload of B)
        run_blocked_host(g, *small, seed=20)
        run_blocked_host(g, *small, seed=20)
        run_blocked_host(g, [150, 64], [1030, 40], [300, 1100], seed=21)    # K split at 1030; last product chunked
        run_blocked_host(g, [64, 30], [4097, 10], [40], seed=22)            # K split at 4097
        run_blocked_host(g, [66], [1030], [1500], seed=23)                  # one product: first and last
    finally:
        lib.mb_shutdown(ctx)


# (rows, k, n) with 1 MiB chunks: 128-row chunks for max(k, n) = 1000; 384-row chunks at max(k, n) = 300, whether k or
# n is the larger; every case more chunks than the 3 ring slots, and rows not a multiple of 128
ROWSHARD = [(1000, 1000, 300), (2000, 100, 300), (2000, 300, 100)]


@pytest.mark.parametrize("dims", ROWSHARD, ids=["x".join(map(str, d)) for d in ROWSHARD])
def test_matmul_rowsharded_host(gpu, dims, monkeypatch):
    lib, ctx = gpu
    monkeypatch.setenv("MARLIN_B200_ROWSHARD_CHUNK_MIB", "1")
    rows, k, n = dims
    chunk = max(128, (2 ** 20 // (8 * max(k, n))) // 128 * 128)
    nchunks = -(-rows // chunk)
    assert nchunks > 3
    A, B, _, want = case(rows, k, n, seed=3)
    Ar, Bc = np.ascontiguousarray(A), np.asfortranarray(B)

    def fn():
        Cm = np.full((rows, n), np.nan)
        nat.check(lib.mb_matmul_rowsharded_host(ctx, Ar.ctypes.data_as(C.c_void_p), rows, k, Bc.ctypes.data_as(C.c_void_p),
                                                n, Cm.ctypes.data_as(C.c_void_p)))
        return Cm

    got, names, launches = profiled(gpu, fn)
    only(names, form(DMMA, 1, 0))
    assert launches == nchunks
    xg.assert_exact(got, want, f"rowsharded host {dims}")


def test_matmul_rowsharded_device(gpu):
    """mb_matmul_rowsharded on device views: row-major A and C (transposed views), column-major B."""
    lib, ctx = gpu
    rows, k, n = ROWSHARD[0]
    A, B, _, want = case(rows, k, n, seed=3)

    def fn():
        sa, sb = Stored(A.T, F64), Stored(B, F64)
        sc = Stored(np.full((n, rows), np.nan), F64)
        ha, hb, hc = sa.block(gpu, True), sb.block(gpu), sc.block(gpu, True)
        nat.check(lib.mb_matmul_rowsharded(ctx, ha, hb, hc))
        nat.check(lib.mb_synchronize(ctx))
        got, clean = sc.read()
        return got.T, clean

    (got, clean), names, launches = profiled(gpu, fn)
    only(names, form(DMMA, 1, 0))
    assert launches == 1 and clean
    xg.assert_exact(got, want, "rowsharded device")


# ====================================================================================================== f. Gramian
# (n, m, layout, split-K): n = 1024 over m = 8192 and n = 333 split K (DESIGN 3.7); n = 2817 (23 tile rows) and 2816
# (22: the triangle is below two waves, but no split fills the last wave 1 % better) run one pass, mirrored in place
GRAMIANS = [(1024, 8192, "columns", True), (333, 20000, "rows", True), (2817, 2048, "columns", False),
            (2816, 2048, "rows", False)]


@pytest.mark.parametrize("gram", GRAMIANS, ids=[f"{g[0]}x{g[1]}-{g[2]}" for g in GRAMIANS])
def test_gramian(gpu, gram):
    """G = A^T A of a column-major block, or X X^T of a row shard (the transposed view of X = A^T), against the exact
    product; G is exactly symmetric, since every split partial is exact and so is their sum."""
    import torch
    lib, ctx = gpu
    n, m, layout, split = gram
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ws = lib.mb_gramian_workspace_bytes(n, m, sms)
    assert (ws > 0) == split, (gram, ws)
    A = xg.gram_operand(np.random.default_rng(n + m), m, n)
    want = xg.reference(A.T, A)

    def fn():
        sa = Stored(A, F64) if layout == "columns" else Stored(A.T, F64, ld=even(n))
        sg = Stored(np.full((n, n), np.nan), F64, ld=even(n) + 2)
        ha = sa.block(gpu, layout == "rows")
        hg = sg.block(gpu)
        nat.check(lib.mb_block_gramian(ctx, ha, hg))
        nat.check(lib.mb_synchronize(ctx))
        lib.mb_block_free(ctx, ha)
        lib.mb_block_free(ctx, hg)
        return sg.read()

    (G, clean), names, launches = profiled(gpu, fn)
    trans = layout == "columns"
    only(names, form("syrk_f64_dmma16x8_kernel", trans, not trans), "gram_reduce_mirror_kernel")
    assert launches == 2 and clean
    xg.assert_exact(G, want, f"Gramian {gram}")
    assert np.array_equal(G, G.T)


# ============================================================================================= g. the Python API
def test_block_matrix_multiply_ragged():
    """BlockMatrix.multiply on a 3 x 3 x 3 grid of 334 / 332-row, 234 / 232-k and 167 / 166-column integer blocks: one
    grouped launch, == the host product."""
    import marlin_b200 as mb
    from marlin_b200.matrix.block import BlockID
    from marlin_b200.matrix.block_matrix import BlockMatrix
    from marlin_b200.matrix.sub_matrix import SubMatrix
    rt = mb.Runtime.get()
    A, B, _, want = case(1000, 700, 500, seed=4)
    rows, ks, cols = [0, 334, 668, 1000], [0, 234, 468, 700], [0, 167, 334, 500]
    Am = BlockMatrix([(BlockID(i, kk), SubMatrix(A[rows[i]:rows[i + 1], ks[kk]:ks[kk + 1]])) for i in range(3) for kk in range(3)],
                     1000, 700, 3, 3)
    Bm = BlockMatrix([(BlockID(kk, j), SubMatrix(B[ks[kk]:ks[kk + 1], cols[j]:cols[j + 1]])) for kk in range(3) for j in range(3)],
                     700, 500, 3, 3)

    def fn():
        res = Am.multiply(Bm)
        rt.sync_stream()
        return res

    res, names, launches = profiled((rt.lib, rt.ctx), fn)
    only(names, GROUPED)
    assert launches == 1
    xg.assert_exact(res.toBreeze(), want, "BlockMatrix.multiply")


def test_dense_vec_matrix_multiply_local():
    """DenseVecMatrix.multiply(B: BDM): one DMMA product per row shard, == the host product."""
    import marlin_b200 as mb
    rt = mb.Runtime.get()
    A, B, _, want = case(3000, 512, 300, seed=5)
    D = mb.DenseVecMatrix(list(enumerate(A)))

    def fn():
        res = D.multiply(B)
        rt.sync_stream()
        return res

    res, names, launches = profiled((rt.lib, rt.ctx), fn)
    only(names, form(DMMA, 1, 0))                  # the row-major C as C^T = B^T A^T
    assert launches == 1
    xg.assert_exact(res.toBreeze(), want, "DenseVecMatrix.multiply")

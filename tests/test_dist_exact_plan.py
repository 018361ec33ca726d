"""No GPU: every case of the exact multi-GPU multiply tests (tests/dist_exact_cases.py) sits where it claims to.

The fast-path decision of mb_matmul_blocked_dist and the feasibility checks of mb_matmul_blocked_dist_host are restated
here from the plan (the exported host logic mb_dist_plan) and the tile shapes, and every case is checked against them:
at a limit, one past it, on the path it asserts, and with launch counts that tell the two paths apart on every rank.
The data bound of every case is proved with exact_gemm.check_bound, and half_cols / bands_of are checked on the widths
the cases use against a direct restatement."""
import math
import zlib

import numpy as np
import pytest

from tests import dist_exact_cases as dc
from tests import exact_gemm as xg

DEVICE_CASES = dc.DEVICE + dc.FRESH + dc.QUEUED


# ------------------------------------------------------------------------------------------------ the plan, restated
def product_rank(seq, P, world):
    return seq * world // P if P >= world else seq


def holders(m, k, n, world):
    """Per C tile (i * n + j): the ranks holding a partial of it, in kk order of first appearance."""
    P = m * k * n
    out = []
    for t in range(m * n):
        h = []
        for kk in range(k):
            r = product_rank(t * k + kk, P, world)
            if r not in h:
                h.append(r)
        out.append(h)
    return out


def c_tiles_of(m, k, n, world, r):
    """[(id, i, j, kks)] of the C tiles rank r computes partials of, in (i, j) order."""
    P = m * k * n
    out = []
    for t in range(m * n):
        kks = [kk for kk in range(k) if product_rank(t * k + kk, P, world) == r]
        if kks:
            out.append((t, t // n, t % n, kks))
    return out


def operand_counts(k, cs):
    a = {(i, kk) for _, i, _, kks in cs for kk in kks}
    b = {(kk, j) for _, _, j, kks in cs for kk in kks}
    return len(a), len(b)


def half_cols(N):
    return min(N, max(128, (N // 2 + 127) // 128 * 128))


def bands_of(extent, most):
    nb = most if extent >= 1024 else 1
    band = ((extent + nb - 1) // nb + 127) // 128 * 128
    return band, (extent + band - 1) // band


def plain(layout, rows):
    """Does the fast path accept a tile in this layout?  A packed tile's leading dimension is its row count."""
    return rows % 2 == 0 if layout == "" else dc.VIEWS[layout]


def fast_path(case):
    """mb_matmul_blocked_dist's verdict for the whole call, the same on every rank."""
    m, k, n = case.grid
    fast = case.dtype == "f64" and k <= dc.G2_MAX_SEG and not case.slow
    a_view, b_view = dict(case.a_view), dict(case.b_view)
    fast = fast and all(plain(a_view.get(t, ""), case.rows[t // k]) for t in range(m * k))
    fast = fast and all(plain(b_view.get(t, ""), case.ks[t // n]) for t in range(k * n))
    h = holders(m, k, n, case.world)
    # only C tiles with two or more holders are published, and only published tiles are checked
    c_plain = {"": None, "even": True, "odd": False}[case.c_view]
    fast = fast and all(case.rows[t // n] % 2 == 0 if c_plain is None else c_plain for t in range(m * n) if len(h[t]) > 1)
    for r in range(case.world):
        cs = c_tiles_of(m, k, n, case.world, r)
        na, nb = operand_counts(k, cs)
        fast = fast and na <= dc.G2_MAX_OPS and nb <= dc.G2_MAX_OPS and 2 * len(cs) <= dc.G2_MAX_ENTRIES
    pairs = {}
    for t in range(m * n):
        if len(h[t]) == 2:
            key = tuple(sorted(h[t]))
            pairs[key] = pairs.get(key, 0) + 1
    return fast and all(v <= dc.MAX_PAIR for v in pairs.values())


def fast_launches(case, r):
    """Launches rank r makes on the fast path: the first grouped launch (halves the peers reduce, plain tiles), the
    second (halves reduced here) — each only if it has entries — and one add per staged partial it owns."""
    m, k, n = case.grid
    h = holders(m, k, n, case.world)
    l0 = l2 = adds = 0
    for t, i, j, kks in c_tiles_of(m, k, n, case.world, r):
        N = case.cols[j]
        if len(h[t]) == 2:
            owner = h[t][0] == r
            if owner:
                l0 += N > half_cols(N)
                l2 += 1
            else:
                l0 += 1
                l2 += N > half_cols(N)
        else:
            l0 += 1
            if h[t][0] == r:
                adds += len(h[t]) - 1
    return (l0 > 0) + (l2 > 0) + adds


def general_min_launches(case, r):
    """The fewest launches rank r makes on the general path: one per C tile whose every kk is here, one per product
    otherwise, and one add per staged partial it owns."""
    m, k, n = case.grid
    h = holders(m, k, n, case.world)
    out = 0
    for t, i, j, kks in c_tiles_of(m, k, n, case.world, r):
        out += 1 if len(kks) == k else len(kks)
        if h[t][0] == r:
            out += len(h[t]) - 1
    return out


# ------------------------------------------------------------------------------------------------ the host entry, restated
def host_homes(case):
    if case.a_home:
        return list(case.a_home), list(case.b_home)
    return None


def host_verdict(case):
    """The first feasibility check of mb_matmul_blocked_dist_host that fails ("" = feasible), in the entry's order."""
    m, k, n = case.grid
    if k > dc.G2_MAX_SEG:
        return "k"
    homes = host_homes(case)
    total = m * k + k * n
    ups = [0] * case.world
    if homes:
        for hm in homes[0] + homes[1]:
            ups[hm] += 1
    else:                                               # mb_dist_host_homes spreads the uploads as evenly as it can
        ups = [math.ceil(total / case.world)] + [0] * (case.world - 1)
    if max(ups) > dc.UP_SLOTS:
        return "uploads"
    h = holders(m, k, n, case.world)
    if any(len(x) > 2 for x in h):
        return "holders"
    for r in range(case.world):
        cs = c_tiles_of(m, k, n, case.world, r)
        na, nb = operand_counts(k, cs)
        subs, pair = 0, {}
        for t, i, j, kks in cs:
            s = bands_of(case.rows[i], dc.MAX_BANDS)[1] * bands_of(case.cols[j], dc.MAX_BANDS)[1]
            subs += s
            if len(h[t]) == 2:
                peer = h[t][1] if h[t][0] == r else h[t][0]
                pair[peer] = pair.get(peer, 0) + s
        if na > dc.G2_MAX_OPS or nb > dc.G2_MAX_OPS or subs > dc.G2_MAX_ENTRIES:
            return "subs"
        if any(v > dc.SUB_SLOTS for v in pair.values()):
            return "shared_subs"
    return ""


def host_subs(case, r):
    m, k, n = case.grid
    return sum(bands_of(case.rows[i], dc.MAX_BANDS)[1] * bands_of(case.cols[j], dc.MAX_BANDS)[1]
               for _, i, j, _ in c_tiles_of(m, k, n, case.world, r))


# ------------------------------------------------------------------------------------------------ tests
def test_plan_restatement_matches_mb_dist_plan():
    """The restated product -> rank map and C owners are those of the exported host logic."""
    import ctypes as C
    nat = pytest.importorskip("marlin_b200._native")
    try:
        lib = nat.load(build_if_missing=False)
    except Exception as e:                             # the library is built by build(); nothing here needs a GPU
        pytest.skip(f"library not built: {e}")
    grids = {(c.grid, c.world) for c in dc.CASES} | {((m, k, n), w) for m in (1, 2, 3) for k in (1, 2, 5) for n in (1, 4) for w in (2, 3, 5)}
    for (m, k, n), world in sorted(grids):
        pr = (C.c_int32 * (m * k * n))()
        co = (C.c_int32 * (m * n))()
        assert lib.mb_dist_plan(m, k, n, world, pr, co) == 0
        for i in range(m):
            for j in range(n):
                for kk in range(k):
                    seq = i * n * k + j * k + kk
                    assert pr[seq] == product_rank(seq, m * k * n, world)
        assert list(co) == [h[0] for h in holders(m, k, n, world)]


@pytest.mark.parametrize("case", DEVICE_CASES, ids=lambda c: c.name)
def test_device_case_takes_its_path_and_the_launch_count_says_which(case):
    assert fast_path(case) == (case.path == "fast"), f"{case.name} is built for the {case.path} path"
    for r in range(case.world):
        assert 1 <= fast_launches(case, r) <= case.fast_max < general_min_launches(case, r), \
            (case.name, r, fast_launches(case, r), general_min_launches(case, r))


def _limit_value(case, limit):
    """The quantity `limit` names on the rank where it is largest, and the limit itself."""
    m, k, n = case.grid
    per_rank = [c_tiles_of(m, k, n, case.world, r) for r in range(case.world)]
    if limit == "k":
        return k, dc.G2_MAX_SEG
    if limit == "a_ops":
        return max(operand_counts(k, cs)[0] for cs in per_rank), dc.G2_MAX_OPS
    if limit == "b_ops":
        return max(operand_counts(k, cs)[1] for cs in per_rank), dc.G2_MAX_OPS
    if limit == "entries":
        return max(2 * len(cs) for cs in per_rank), dc.G2_MAX_ENTRIES
    raise KeyError(limit)


@pytest.mark.parametrize("case", [c for c in dc.DEVICE if c.limit and c.limit != "plain"], ids=lambda c: c.name)
def test_device_limit_cases_sit_at_or_one_past_their_limit(case):
    value, limit = _limit_value(case, case.limit)
    step = 2 if case.limit == "entries" else 1           # two entries per C tile: 32 / 33 tiles are 64 / 66 entries
    assert value == (limit if case.side == "at" else limit + step), (case.name, value, limit)
    # every other limit is met: the case crosses its own limit only
    for other in {"k", "a_ops", "b_ops", "entries"} - {case.limit}:
        v, lim = _limit_value(case, other)
        assert v <= lim, (case.name, other, v, lim)


def test_plain_limit_cases_differ_from_the_at_case_by_one_layout():
    at = [c for c in dc.CASES if getattr(c, "limit", "") == "plain" and c.side == "at"]
    past = [c for c in dc.CASES if getattr(c, "limit", "") == "plain" and c.side == "past"]
    assert at and past
    layouts = {v for c in past for _, v in c.a_view + c.b_view} | {c.c_view for c in past if c.c_view}
    assert layouts == {"off8", "odd_ld", "T", "odd"}                   # 8-byte offset, odd ld (A and C), transposed
    for c in past:
        twin = next(a for a in at if (a.grid, a.rows, a.ks) == (c.grid, c.rows, c.ks))
        assert fast_path(twin) and not fast_path(c)


def test_fused_pair_and_shared_sub_block_limits_are_unreachable():
    """MAX_PAIR (fused tiles per rank pair) and SUB_SLOTS (shared host sub-blocks per pair) cannot be reached: products
    are dealt to ranks in contiguous seq ranges and a C tile's products are contiguous, so a tile with exactly two
    holders straddles the boundary between two consecutive ranks, and each boundary is crossed by one tile.  So no
    test can stand at or past these limits; this proves it over every small plan."""
    for world in range(2, 7):
        for m in range(1, 6):
            for k in range(1, 8):
                for n in range(1, 6):
                    h = holders(m, k, n, world)
                    pairs = {}
                    for x in h:
                        assert x == list(range(x[0], x[0] + len(x)))          # consecutive ranks
                        if len(x) == 2:
                            pairs[tuple(x)] = pairs.get(tuple(x), 0) + 1
                    assert all(v == 1 for v in pairs.values())
    # one shared tile per pair holds at most MAX_BANDS^2 sub-blocks
    assert dc.MAX_BANDS ** 2 < dc.SUB_SLOTS and 1 < dc.MAX_PAIR


@pytest.mark.parametrize("case", dc.HOST, ids=lambda c: c.name)
def test_host_case_feasibility(case):
    verdict = host_verdict(case)
    if case.error:
        assert verdict == case.limit or (case.name == "k16" and verdict == "uploads"), (case.name, verdict)
    else:
        assert verdict == "", (case.name, verdict)
    if case.limit == "uploads":
        ups = max(np.bincount(list(case.a_home) + list(case.b_home)))
        assert ups == (dc.UP_SLOTS if case.side == "at" else dc.UP_SLOTS + 1)
    if case.limit == "subs":
        most = max(host_subs(case, r) for r in range(case.world))
        assert most == (dc.G2_MAX_ENTRIES if case.side == "at" else dc.G2_MAX_ENTRIES + 1)
    if case.limit == "k":
        assert case.grid[1] == (dc.G2_MAX_SEG if case.side == "at" else dc.G2_MAX_SEG + 1)


def test_host_k_limit_is_shadowed_by_the_upload_limit_on_two_ranks():
    """k = 16 reads 16 A and 16 B tiles at least; two ranks upload at most 2 x UP_SLOTS = 16 of them."""
    assert 2 * dc.G2_MAX_SEG > 2 * dc.UP_SLOTS


def test_every_refused_host_call_is_followed_by_one_that_must_succeed():
    hl = dc.group("host_limits")
    for i, c in enumerate(hl):
        if c.error:
            assert i + 1 < len(hl) and any(not later.error for later in hl[i + 1:i + 3]), c.name
    assert not hl[-1].error


def test_host_checkerboards_cover_1x1_3x3_and_4x4():
    grids = {(bands_of(c.rows[0], 4)[1], bands_of(c.cols[0], 4)[1]) for c in dc.group("host") if c.grid == (1, 2, 1)}
    assert {(1, 1), (3, 3), (4, 4)} <= grids


def test_column_split_and_bands_on_the_case_widths():
    widths = sorted({N for c in dc.group("split") for N in c.cols})
    assert {1, 100, 128, 129, 255, 256, 257, 385} <= set(widths)
    extents = {c.rows[0] for c in dc.group("split")} | {c.cols[0] for c in dc.group("split")}
    assert {1023, 1024, 1025, 1537} <= extents
    # owner [0, half_cols(N)), partner [half_cols(N), N): a multiple of 128 or all of N, never empty on the owner's side
    # (a zero-wide grouped entry is refused), empty on the partner's up to N = 128
    want = {1: 1, 100: 100, 128: 128, 129: 128, 255: 128, 256: 128, 257: 128, 385: 256}
    for N, h in want.items():
        assert half_cols(N) == h, N
    for N in range(1, 2000):
        h = half_cols(N)
        assert 0 < h <= N and (h == N or h % 128 == 0)
        assert (N - h == 0) == (N <= 128)
        assert N // 2 <= h < N // 2 + 128
    want_bands = {1023: (1023 // 128 * 128 + 128, 1), 1024: (256, 4), 1025: (384, 3), 1537: (512, 4)}
    for e, (band, nb) in want_bands.items():
        assert bands_of(e, 4) == (band, nb), e
    assert 1537 - 3 * 512 == 1                              # a one-wide last band
    for e in range(1, 5000):
        band, nb = bands_of(e, 4)
        assert band % 128 == 0 and (nb - 1) * band < e <= nb * band and nb <= 4
        assert nb == 1 or e >= 1024


def _operands(case, rep=0):
    """The data of the rank program, without ctypes: same generator, same seed."""
    from tests import dist_exact_worker as w
    return w.make_operands(case, rep)


@pytest.mark.parametrize("case", [c for c in dc.CASES if not getattr(c, "error", "")], ids=lambda c: c.name)
def test_case_data_is_exact_in_every_order(case):
    reps = getattr(case, "reps", 1)
    for rep in range(reps):
        A, B, ref = _operands(case, rep)
        assert A.shape == (sum(case.rows), sum(case.ks)) and B.shape == (sum(case.ks), sum(case.cols))
        if getattr(case, "dtype", "f64") == "bf16":
            assert np.abs(A).max() <= 256 and np.abs(B).max() <= 256
            assert A.shape[1] * 256 * 256 < 2 ** 24
            assert np.array_equal(ref, A @ B)
            continue
        fa, fb = np.where(np.isfinite(A), A, 0), np.where(np.isfinite(B), B, 0)
        w = xg.check_bound(fa, fb)
        assert w >= xg.TWO52                                  # the results use the whole significand
        if not getattr(case, "special", False):
            assert np.array_equal(ref, A @ B)
    # fresh operands per call: no two calls of a case see the same data
    if reps > 1:
        assert not np.array_equal(_operands(case, 0)[0], _operands(case, 1)[0])


def test_special_values_reach_the_non_owner_segments_and_the_classes_follow_ieee():
    case = dc.by_name("nan_inf")
    A, B, ref = _operands(case)
    m, k, n = case.grid
    h = holders(m, k, n, case.world)[0]
    assert h == [0, 1]
    kk_partner = c_tiles_of(m, k, n, case.world, 1)[0][3]
    lo = sum(case.ks[:kk_partner[0]])
    hi = sum(case.ks[:kk_partner[-1] + 1])
    bad_cols = np.where(~np.isfinite(A).all(axis=0))[0]
    bad_rows = np.where(~np.isfinite(B).all(axis=1))[0]
    assert len(bad_cols) and all(lo <= c < hi for c in bad_cols)
    assert len(bad_rows) and all(lo <= r < hi for r in bad_rows)
    assert np.isnan(A).sum() == 1 and np.isinf(A).sum() == 1 and np.isinf(B).sum() == 1
    jc = int(np.where(np.isinf(B).any(axis=0))[0][0])
    assert jc < half_cols(case.cols[0])                          # the +Inf column is reduced by the owner
    with np.errstate(invalid="ignore"):
        direct = A @ B                                          # numpy's classes, for comparison
    assert np.array_equal(np.isnan(ref), np.isnan(direct))
    assert np.array_equal(np.isposinf(ref), np.isposinf(direct)) and np.array_equal(np.isneginf(ref), np.isneginf(direct))
    assert np.isnan(ref).any() and np.isposinf(ref).any() and np.isneginf(ref).any()


def test_fresh_group_alternates_plans_and_grows_then_reuses_staging():
    fresh, queued = dc.group("fresh"), dc.group("queued")
    assert len(fresh) >= 6 and len(queued) >= 5
    assert any(c.slow for c in fresh)
    grids = [c.grid for c in fresh]
    assert all(a != b for a, b in zip(grids, grids[1:])) or len(set(grids)) >= 2
    # the staging slot a call needs: the fused tile's larger half (even rows) per direction
    def need(c):
        m, k, n = c.grid
        h = holders(m, k, n, c.world)
        out = 0
        for t in range(m * n):
            if len(h[t]) == 2:
                N = c.cols[t % n]
                M = c.rows[t // n] + c.rows[t // n] % 2
                out = max(out, M * max(half_cols(N), N - half_cols(N)) * 8)
        return out
    needs = [need(c) for c in fresh]
    grow = needs.index(max(needs))
    assert 0 < grow < len(fresh) - 2 and all(x < needs[grow] for x in needs[grow + 1:])
    assert len({c.name for c in queued}) == len(queued)


def test_seeds_differ_between_cases():
    seeds = [zlib.crc32(f"{c.group}/{c.name}/0".encode()) for c in dc.CASES]
    assert len(set(seeds)) == len(seeds)

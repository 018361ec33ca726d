"""StandardNormalGenerator(mean, variance) (utils/RandomDataGenerator.scala:70-82) restated for the tests, twice:

- XORShiftNormal: java.util.Random.nextGaussian (als_oracle.JavaRandom's) over XORShiftRandom.next (:113-131), one value
  at a time, the way XORShiftRandom overrides `next` under the JDK's own nextDouble and nextGaussian;
- normal_stream: the same values vectorised in numpy, from the partition's uniform stream (the `oracle` package's
  UniformGenerator restatement: u = nextDouble), the polar step and fdlibm's log on int64 views.  numpy never contracts a
  multiply and an add, so every operation is rounded separately, as on the JVM.

normal_stream also returns 2A, the nextDouble positions the values consumed (A = the last attempt used plus one), and how
often each branch of fdlibm's log was taken.
"""
from __future__ import annotations

import math

import numpy as np

from tests import als_oracle as ao

M64 = (1 << 64) - 1
LN2_HI, LN2_LO = 6.93147180369123816490e-01, 1.90821492927058770002e-10
LG1, LG2, LG3, LG4, LG5, LG6, LG7 = ao._LG

# fdlibm log branches nextGaussian's s in (0, 1) can reach.  "small_f0" (f == 0: s an exact power of two) is reachable
# but needs s to land exactly on a power of two, about one attempt in 2^52; "small_f0" with k == 0 would need s == 1.
BRANCHES = ("small_f0", "small_k0", "small_k", "pos_k0", "pos_k", "neg_k0", "neg_k")


def sd_of(variance: float) -> float:
    """math.sqrt(variance) on the JVM: NaN for a negative or NaN variance."""
    with np.errstate(invalid="ignore"):
        return float(np.sqrt(np.float64(variance)))


class XORShiftNormal(ao.JavaRandom):
    """generator.copy(); setSeed(p); nextValue() ... for StandardNormalGenerator(mean, variance)."""

    def __init__(self, partition_seed: int, mean: float = 0.0, variance: float = 1.0):
        from oracle import reference_model as rm
        super().__init__(0)
        self.seed = rm.hash_seed(partition_seed) & M64
        self.mean, self.sd = float(mean), sd_of(variance)

    def next(self, bits: int) -> int:
        s = self.seed
        s ^= (s << 21) & M64
        s ^= s >> 35
        s ^= (s << 4) & M64
        self.seed = s
        return s & ((1 << bits) - 1)

    def next_value(self) -> float:
        return self.mean + self.sd * self.next_gaussian()


def fdlibm_log_vec(x: np.ndarray, counts: dict | None = None) -> np.ndarray:
    """fdlibm e_log.c for positive normal doubles x < 1 (als_oracle.fdlibm_log element by element), on int64 views.
    counts (optional) is incremented per branch taken (BRANCHES)."""
    x = np.ascontiguousarray(x, dtype=np.float64)
    bits = x.view(np.int64)
    hx = bits >> 32
    assert ((hx >= 0x00100000) & (hx < 0x3FF00000)).all()
    k = (hx >> 20) - 1023
    hx = hx & 0x000FFFFF
    i = (hx + 0x95F64) & 0x100000
    xn = (((hx | (i ^ 0x3FF00000)) << 32) | (bits & 0xFFFFFFFF)).view(np.float64)
    k = k + (i >> 20)
    f = xn - 1.0
    dk = k.astype(np.float64)
    k0 = k == 0
    small = (0x000FFFFF & (2 + hx)) < 3
    small_f0 = small & (f == 0.0)
    res = np.empty_like(f)
    # |f| < 2^-20
    r_small = f * f * (0.5 - 0.33333333333333333 * f)
    res_small = np.where(k0, f - r_small, dk * LN2_HI - ((r_small - dk * LN2_LO) - f))
    res_f0 = np.where(k0, 0.0, dk * LN2_HI + dk * LN2_LO)
    # the rest
    s = f / (2.0 + f)
    z = s * s
    w = z * z
    t1 = w * (LG2 + w * (LG4 + w * LG6))
    t2 = z * (LG1 + w * (LG3 + w * (LG5 + w * LG7)))
    ii = (hx - 0x6147A) | (0x6B851 - hx)
    R = t2 + t1
    hfsq = 0.5 * f * f
    res_pos = np.where(k0, f - (hfsq - s * (hfsq + R)), dk * LN2_HI - ((hfsq - (s * (hfsq + R) + dk * LN2_LO)) - f))
    res_neg = np.where(k0, f - s * (f - R), dk * LN2_HI - ((s * (f - R) - dk * LN2_LO) - f))
    pos = ~small & (ii > 0)
    neg = ~small & ~(ii > 0)
    res[:] = np.where(pos, res_pos, res_neg)
    res[small] = res_small[small]
    res[small_f0] = res_f0[small_f0]
    if counts is not None:
        for name, mask in (("small_f0", small_f0), ("small_k0", small & ~small_f0 & k0), ("small_k", small & ~small_f0 & ~k0),
                           ("pos_k0", pos & k0), ("pos_k", pos & ~k0), ("neg_k0", neg & k0), ("neg_k", neg & ~k0)):
            counts[name] = counts.get(name, 0) + int(mask.sum())
    return res


def _uniforms(partition_seed: int, first: int, n: int) -> np.ndarray:
    """nextDouble positions [first, first + n) of the partition's stream (a far start by jump-ahead)."""
    from oracle import reference_model as rm
    if first < (1 << 22):
        return rm.uniform_stream(partition_seed, first, n)
    return rm.uniform_stream_far(partition_seed, first, n)


def accepted_attempts(partition_seed: int, attempts: int, first: int = 0) -> np.ndarray:
    """Which of attempts [first, first + attempts) of the partition's polar method are accepted (bool array)."""
    u = _uniforms(partition_seed, 2 * first, 2 * attempts)
    v1, v2 = 2 * u[0::2] - 1, 2 * u[1::2] - 1
    s = v1 * v1 + v2 * v2
    return (s < 1) & (s != 0)


def normal_stream(partition_seed: int, n: int, mean: float = 0.0, variance: float = 1.0, chunk: int = 1 << 22,
                  first_attempt: int = 0):
    """(the first n values of StandardNormalGenerator(mean, variance) after setSeed(partition_seed), 2A, branch counts).
    first_attempt > 0: the values of the attempts from that one on (they follow value 2 * (accepted attempts before it))."""
    pairs = (n + 1) // 2
    if pairs == 0:
        return np.zeros(0), 0, {}
    v1s, v2s, ss, idx = [], [], [], []
    got, a0 = 0, first_attempt
    while got < pairs:
        want = max(chunk, int(math.ceil((pairs - got) * 4 / math.pi * 1.01)) + 64)
        u = _uniforms(partition_seed, 2 * a0, 2 * want)
        v1, v2 = 2 * u[0::2] - 1, 2 * u[1::2] - 1
        s = v1 * v1 + v2 * v2
        ok = (s < 1) & (s != 0)
        v1s.append(v1[ok]); v2s.append(v2[ok]); ss.append(s[ok]); idx.append(np.nonzero(ok)[0] + a0)
        got += int(ok.sum())
        a0 += want
    v1, v2, s, idx = (np.concatenate(a)[:pairs] for a in (v1s, v2s, ss, idx))
    counts: dict = {}
    mult = np.sqrt(-2 * fdlibm_log_vec(s, counts) / s)
    g = np.empty(2 * pairs)
    g[0::2] = v1 * mult
    g[1::2] = v2 * mult
    with np.errstate(invalid="ignore"):
        vals = np.float64(mean) + np.float64(sd_of(variance)) * g[:n]
    return vals, 2 * (int(idx[-1]) + 1), counts


def budget_tiles(pairs: int, tile: int) -> int:
    """Tiles mb_fill_normal counts for a deficit of `pairs` pairs (MB_NORMAL_TILE_ATTEMPTS in include/marlin_b200.h)."""
    return -(-math.ceil(pairs * 4.0 / 3.141592653589793) // tile)


def counting_rounds(partition_seed: int, n: int, tile: int) -> int:
    """How many counting rounds mb_fill_normal runs for n values: the first budget, then more while it falls short."""
    pairs = (n + 1) // 2
    counted, total, rounds = 0, 0, 0
    add = budget_tiles(pairs, tile)
    while True:
        total += int(accepted_attempts(partition_seed, add * tile, counted * tile).sum())
        counted += add
        rounds += 1
        if total >= pairs:
            return rounds
        add = budget_tiles(pairs - total, tile)

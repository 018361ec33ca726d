"""The case table of the exact-integer tests of the multi-GPU block multiply (mb_matmul_blocked_dist and
mb_matmul_blocked_dist_host): read by the rank program (tests/dist_exact_worker.py), by the GPU tests that start it
(tests/test_gpu_dist_cabi.py) and by the plan test that proves, without a GPU, that every case sits where it claims to
(tests/test_dist_exact_plan.py).

A device case names a block grid (m, k, n), the block extents, the owner of every operand tile, how each tile is laid
out in device memory and the path the call must take:
  "fast"    : plain fp64 tiles, every rank's share within one grouped launch, C tiles with two holders fused
              (reduce-scatter in the GEMM epilogues): at most `fast_max` kernel launches on every rank;
  "general" : per-tile launches and staged partials: more than `fast_max` launches on every rank.
The plan test shows that the two launch-count ranges are disjoint on every rank of every case, so the count the rank
program reads from mb_launch_count names the path that ran.

A host case drives mb_matmul_blocked_dist_host; `error` is a piece of the message every rank must return with
MB_ERR_UNSUPPORTED, or "" when the call must succeed.  Feasibility limits are only tested where every rank decides them
before any exchange.
"""
from __future__ import annotations

from dataclasses import dataclass

# The limits of csrc/dist.cu and csrc/gemm_f64.h the cases are built around.
G2_MAX_SEG = 16         # k segments per grouped entry
G2_MAX_OPS = 32         # distinct A (and B) operand tiles per grouped launch
G2_MAX_ENTRIES = 64     # entries per grouped launch
MAX_PAIR = 8            # fused C tiles per rank pair and call
MAX_BANDS = 4           # readiness bands per operand tile
UP_SLOTS = 8            # host entry: tiles one rank uploads
SUB_SLOTS = 64          # host entry: shared sub-blocks per rank pair


@dataclass(frozen=True)
class Case:
    name: str
    group: str
    grid: tuple                      # (m, k, n)
    rows: tuple                      # row_len[i]
    ks: tuple                        # k_len[kk]
    cols: tuple                      # col_len[j]
    path: str = "fast"               # "fast" | "general"
    limit: str = ""                  # the limit the case tests ("" = none)
    side: str = ""                   # "at" | "past" the limit
    a_view: tuple = ()               # ((A tile, layout), ...): layouts in VIEWS
    b_view: tuple = ()
    c_view: str = ""                 # layout of every C tile the owner holds: "" packed, "even" / "odd" parent slice
    dtype: str = "f64"               # "f64" | "bf16" (fp32 C)
    special: bool = False            # NaN / Inf operands on the rank that does not own the C tile
    slow: bool = False               # MARLIN_B200_DIST_SLOW=1 for this call
    world: int = 2
    fast_max: int = 2                # most launches a rank makes on the fast path (grouped launches + staged adds)
    a_owner: tuple = ()              # () = (t + 1) % world: every tile a product reads is pulled from the peer
    b_owner: tuple = ()

    def owners(self):
        m, k, n = self.grid
        a = self.a_owner or tuple((t + 1) % self.world for t in range(m * k))
        b = self.b_owner or tuple((t + 1) % self.world for t in range(k * n))
        return a, b


# Layouts of an operand tile on its owner, and whether the fast path accepts it ("plain": fp64, not transposed, even
# leading dimension, 16-byte aligned first element).  A packed tile ("") is plain when its row count is even.
VIEWS = {
    "off16": True,       # rows [2, 2 + r) of a parent with an even leading dimension: offset 16 bytes
    "off8": False,       # rows [1, 1 + r) of a parent with an even leading dimension: offset 8 bytes
    "odd_ld": False,     # rows [0, r) of a parent with an odd leading dimension
    "T": False,          # the transpose of a packed c x r block, handed out as a transposed view
}


@dataclass(frozen=True)
class HostCase:
    name: str
    group: str
    grid: tuple
    rows: tuple
    ks: tuple
    cols: tuple
    limit: str = ""
    side: str = ""
    error: str = ""                  # expected message part of MB_ERR_UNSUPPORTED on every rank ("" = must succeed)
    a_home: tuple = ()               # () = mb_dist_host_homes
    b_home: tuple = ()
    reps: int = 2
    world: int = 2


def _u(n, v):
    return (v,) * n


DEVICE = [
    # ---- path limits, device entry ----
    Case("k16", "limits", (1, 16, 1), (40,), _u(16, 12), (200,), "fast", "k", "at"),
    Case("k17", "limits", (1, 17, 1), (40,), _u(17, 12), (200,), "general", "k", "past"),
    Case("a_ops32", "limits", (21, 3, 1), _u(21, 24), (16, 16, 16), (40,), "fast", "a_ops", "at"),
    Case("a_ops33", "limits", (22, 3, 1), _u(22, 24), (16, 16, 16), (40,), "general", "a_ops", "past"),
    Case("b_ops32", "limits", (1, 3, 21), (40,), (16, 16, 16), _u(21, 24), "fast", "b_ops", "at"),
    Case("b_ops33", "limits", (1, 3, 22), (40,), (16, 16, 16), _u(22, 24), "general", "b_ops", "past"),
    Case("c_tiles32", "limits", (8, 1, 8), _u(8, 16), (24,), _u(8, 20), "fast", "entries", "at"),
    Case("c_tiles33", "limits", (6, 1, 11), _u(6, 16), (24,), _u(11, 20), "general", "entries", "past"),
    Case("plain_a_off16", "limits", (1, 6, 1), (96,), _u(6, 20), (260,), "fast", "plain", "at", a_view=((0, "off16"),)),
    Case("a_off8", "limits", (1, 6, 1), (96,), _u(6, 20), (260,), "general", "plain", "past", a_view=((0, "off8"),)),
    Case("a_odd_ld", "limits", (1, 6, 1), (96,), _u(6, 20), (260,), "general", "plain", "past", a_view=((1, "odd_ld"),)),
    Case("b_transposed", "limits", (1, 6, 1), (96,), _u(6, 20), (260,), "general", "plain", "past", b_view=((2, "T"),)),
    # ---- the fused column split (owner [0, half_cols(N)), partner the rest) and the readiness bands ----
    *[Case(f"split_n{N}", "split", (1, 6, 1), (72,), _u(6, 8), (N,)) for N in (1, 100, 128, 129, 255, 256, 257, 385)],
    # (a packed tile's leading dimension is its row count: odd-row A and C tiles live in even-ld parents to stay plain)
    *[Case(f"bands_{M}x{N}", "split", (1, 6, 1), (M,), _u(6, 8), (N,), a_view=tuple((t, "off16") for t in range(6)) if M % 2 else (),
           c_view="even" if M % 2 else "")
      for M, N in ((1023, 1023), (1024, 1024), (1025, 1537), (1537, 1025))],
    # ---- C views: the owner's C tile is a slice of a sentinel-filled parent ----
    Case("c_view_even_ld", "views", (1, 6, 1), (96,), _u(6, 20), (300,), "fast", "plain", "at", c_view="even"),
    Case("c_view_odd_ld", "views", (1, 6, 1), (96,), _u(6, 20), (300,), "general", "plain", "past", c_view="odd"),
    # a C tile with one holder is never published, so its layout does not decide the path: odd ld stays fast
    Case("c_view_odd_ld_unshared", "views", (2, 1, 2), (96, 64), (40,), (150, 33), "fast", c_view="odd", fast_max=1),
    # ---- bf16 tiles: general path, fp32 C ----
    Case("bf16_k_split", "bf16", (1, 6, 1), (70,), _u(6, 40), (90,), "general", dtype="bf16"),
    Case("bf16_ragged", "bf16", (3, 2, 2), (70, 33, 64), (120, 100), (90, 17), "general", dtype="bf16"),
    # ---- special values, landing through the staged partial of the fused tile ----
    Case("nan_inf", "special", (1, 6, 1), (64,), _u(6, 8), (300,), "fast", special=True),
    # ---- three or more holders: staged partials, added by the owner in holder order ----
    Case("holders3_fast", "holders3", (1, 12, 1), (80,), _u(12, 10), (200,), "fast", world=3, fast_max=3),
    Case("holders3_slow", "holders3", (1, 12, 1), (80,), _u(12, 10), (200,), "general", slow=True, world=3, fast_max=3),
]

# One communicator, fresh operands and NaN-refilled C tiles every call, alternating plans: each call is checked before
# the next.  The third call grows the staging buffer; the two after it reuse it; one call takes the staged path.
FRESH = [
    Case("f0_fused", "fresh", (1, 6, 1), (64,), _u(6, 8), (300,)),
    Case("f1_222", "fresh", (2, 2, 2), (64, 40), (20, 20), (150, 130), fast_max=1),
    Case("f2_grow", "fresh", (1, 6, 1), (600,), _u(6, 8), (900,)),
    Case("f3_small", "fresh", (1, 6, 1), (48,), _u(6, 8), (260,)),
    Case("f4_slow", "fresh", (2, 2, 2), (64, 40), (20, 20), (150, 130), "general", slow=True, fast_max=1),
    Case("f5_222", "fresh", (2, 2, 2), (32, 72), (20, 20), (140, 200), fast_max=1),
    Case("f6_fused", "fresh", (1, 6, 1), (80,), _u(6, 8), (129,)),
]
# Queued without a host synchronisation: distinct operands, distinct C tiles, checked after the last call.
QUEUED = [
    Case("q0", "queued", (1, 6, 1), (64,), _u(6, 8), (300,)),
    Case("q1", "queued", (2, 2, 2), (64, 40), (20, 20), (150, 130), fast_max=1),
    Case("q2", "queued", (1, 6, 1), (72,), _u(6, 8), (257,)),
    Case("q3", "queued", (1, 6, 1), (64,), _u(6, 8), (300,)),
    Case("q4", "queued", (2, 2, 2), (40, 64), (20, 20), (130, 150), fast_max=1),
    Case("q5", "queued", (1, 6, 1), (100,), _u(6, 8), (128,)),
]

HOST = [
    # checkerboards of (row band x column band) sub-blocks: 1 x 1, 3 x 3, 4 x 4 (and 4 x 4 with a one-wide last band)
    HostCase("host_1x1", "host", (1, 2, 1), (100,), (16, 16), (100,)),
    HostCase("host_4x4", "host", (1, 2, 1), (1024,), (16, 16), (1024,)),
    HostCase("host_3x3", "host", (1, 2, 1), (1025,), (16, 16), (1025,)),
    HostCase("host_1537", "host", (1, 2, 1), (1537,), (16, 16), (1537,)),
    HostCase("host_1023x1025", "host", (1, 2, 1), (1023,), (16, 16), (1025,)),
    HostCase("host_222", "host", (2, 2, 2), (1023, 1025), (16, 16), (1537, 100)),
    # feasibility limits, each one past followed by a call that must succeed on the same communicator
    HostCase("up8", "host_limits", (1, 5, 1), (64,), _u(5, 12), (96,), "uploads", "at",
             a_home=(0, 0, 0, 0, 0), b_home=(0, 0, 0, 1, 1)),
    HostCase("up9", "host_limits", (1, 5, 1), (64,), _u(5, 12), (96,), "uploads", "past", "rank 0 would upload 9 tiles (limit 8)",
             a_home=(0, 0, 0, 0, 0), b_home=(0, 0, 0, 0, 1)),
    HostCase("after_up9", "host_limits", (1, 2, 1), (100,), (16, 16), (100,)),
    HostCase("k17", "host_limits", (1, 17, 1), (40,), _u(17, 4), (40,), "k", "past", "k = 17 > 16"),
    HostCase("after_k17", "host_limits", (1, 2, 1), (64,), (16, 16), (130,)),
    # k = 16 needs 32 uploads, more than two ranks' 2 x 8 slots: the upload limit rejects it first
    HostCase("k16", "host_limits", (1, 16, 1), (40,), _u(16, 4), (40,), "k", "at", "would upload 16 tiles (limit 8)"),
    HostCase("subs64", "host_limits", (3, 1, 3), (1024, 1024, 100), (8,), (1025, 1025, 1024), "subs", "at", reps=1),
    HostCase("subs65", "host_limits", (3, 1, 3), (1024, 1025, 100), (8,), (1025, 1024, 1024), "subs", "past",
             "rank 0's share (65 sub-blocks) does not fit one grouped launch"),
    HostCase("after_subs65", "host_limits", (1, 2, 1), (1025,), (16, 16), (257,)),
]

CASES = DEVICE + FRESH + QUEUED + HOST
GROUPS = sorted({c.group for c in CASES})


def group(name: str):
    out = [c for c in CASES if c.group == name]
    if not out:
        raise KeyError(name)
    return out


def by_name(name: str):
    return next(c for c in CASES if c.name == name)

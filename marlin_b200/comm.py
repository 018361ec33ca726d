"""Placement and exchange planning for the multiply path on G GPUs (one process per GPU).

Marlin replicates A tiles n times and B tiles m times through two Spark shuffles so that partition
`seq = i*n*k + j*k + kk` holds exactly A(i,kk) and B(kk,j), multiplies there, and sums the k partials
per C tile with reduceByKey (matrix/BlockMatrix.scala:159-178).  Here the m*k*n products are mapped
onto ranks, tiles move once over NVLink with grouped NCCL send/recv, and partials that end up on
different ranks are reduced onto the C tile's owner.

Everything in this module is pure planning + torch.distributed plumbing on whatever tensors it is
given (NCCL for CUDA tensors, gloo for the CPU tests); it contains no arithmetic.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Callable, Dict, List, Sequence, Tuple

import torch

Product = Tuple[int, int, int]          # (i, j, kk)


def elem_owner(row: int, col: int, blks_by_col: int, world: int) -> int:
    """Home rank of block (row, col): MatrixElemOpPartitioner partition (rdd/MatrixElemOpPartitioner.scala:16) mod G."""
    return (row * blks_by_col + col) % world


def product_rank(seq: int, num_products: int, world: int) -> int:
    """Rank that runs block product `seq`.  Products are dealt out evenly in contiguous seq ranges, so the
    kk-partials of one C tile (consecutive seq) stay on one rank whenever the ranks get whole C tiles
    (m*n a multiple of G: C-stationary, no reduction traffic); otherwise a kk-group may straddle two ranks
    and that C tile is reduced onto the rank of its kk = 0 partial — an even load beats an idle GPU.
    With fewer C tiles than ranks the k dimension is split across ranks; with G = m*k*n this is the
    reference's identity map partition -> executor."""
    if num_products >= world:
        return (seq * world) // num_products
    return seq


@dataclass
class MultiplyPlan:
    m: int
    k: int
    n: int
    world: int
    products: Dict[int, List[Product]] = field(default_factory=dict)        # rank -> products it computes (seq order)
    a_sends: List[Tuple[int, int, Tuple[int, int]]] = field(default_factory=list)   # (src, dst, (i, kk))
    b_sends: List[Tuple[int, int, Tuple[int, int]]] = field(default_factory=list)   # (src, dst, (kk, j))
    c_owner: Dict[Tuple[int, int], int] = field(default_factory=dict)       # (i, j) -> rank holding the final tile
    c_reduces: List[Tuple[int, int, Tuple[int, int]]] = field(default_factory=list)  # (src, dst, (i, j)) partial -> owner


def plan_multiply(m: int, k: int, n: int, world: int, a_owner: Callable[[int, int], int],
                  b_owner: Callable[[int, int], int]) -> MultiplyPlan:
    plan = MultiplyPlan(m, k, n, world)
    P = m * k * n
    need_a: Dict[Tuple[int, int], set] = {}
    need_b: Dict[Tuple[int, int], set] = {}
    holders: Dict[Tuple[int, int], List[int]] = {}
    for i in range(m):
        for j in range(n):
            for kk in range(k):
                seq = i * n * k + j * k + kk
                r = product_rank(seq, P, world)
                plan.products.setdefault(r, []).append((i, j, kk))
                need_a.setdefault((i, kk), set()).add(r)
                need_b.setdefault((kk, j), set()).add(r)
                h = holders.setdefault((i, j), [])
                if r not in h:
                    h.append(r)
    for (i, kk), ranks in sorted(need_a.items()):
        src = a_owner(i, kk)
        for dst in sorted(ranks):
            if dst != src:
                plan.a_sends.append((src, dst, (i, kk)))
    for (kk, j), ranks in sorted(need_b.items()):
        src = b_owner(kk, j)
        for dst in sorted(ranks):
            if dst != src:
                plan.b_sends.append((src, dst, (kk, j)))
    for key, ranks in sorted(holders.items()):
        plan.c_owner[key] = ranks[0]                 # rank of the kk = 0 partial
        for src in ranks[1:]:
            plan.c_reduces.append((src, ranks[0], key))
    return plan


def exchange(sends: Sequence[Tuple[int, int, object]], local: Dict[object, torch.Tensor],
             alloc: Callable[[object], torch.Tensor], rank: int, group=None) -> Dict[object, torch.Tensor]:
    """Run a list of (src, dst, key) transfers as ONE grouped batch of P2P ops.

    `local[key]` is the tensor to send when this rank is a source; `alloc(key)` returns the receive buffer
    when it is a destination.  Returns {key: received tensor}.  All ranks must call with the same list.
    """
    import torch.distributed as dist
    # gloo moves host memory only: device tensors travel through host copies there (ranks that share one GPU)
    staged = dist.get_backend(group) == "gloo"
    ops = []
    received: Dict[object, torch.Tensor] = {}
    landing: Dict[object, torch.Tensor] = {}
    for (src, dst, key) in sends:
        if src == rank:
            t = local[key]
            ops.append(dist.P2POp(dist.isend, t.cpu() if staged and t.is_cuda else t, dst, group))
        elif dst == rank:
            buf = alloc(key)
            received[key] = buf
            if staged and buf.is_cuda:
                landing[key] = torch.empty(buf.shape, dtype=buf.dtype)
            ops.append(dist.P2POp(dist.irecv, landing.get(key, buf), src, group))
    if ops:
        for req in dist.batch_isend_irecv(ops):
            req.wait()
    for key, host in landing.items():
        received[key].copy_(host)
    return received

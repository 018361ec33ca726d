"""The step plan of the sharded block LU / Cholesky / inverse (marlin_b200.matrix.factorizations.plan_step), checked on
the host: every operation finds its inputs on its rank, nothing moves that need not, and one rank moves nothing."""
import pytest

from marlin_b200 import comm
from marlin_b200.matrix import factorizations as fz

SEQUENCES = {"lu": ["lu"], "cholesky": ["cholesky"], "inverse": ["inverse", "inverse_back"]}


def _initial(algo, nb, world):
    """rank -> keys it holds before the first step: its own blocks of the grid."""
    held = {r: set() for r in range(world)}
    for r in range(nb):
        for c in range(nb):
            if algo != "cholesky" or r >= c:
                held[comm.elem_owner(r, c, nb, world)].add(("A", r, c))
    return held


def _simulate(algo, nb, world):
    held = _initial(algo, nb, world)
    total_sends = 0
    for kind in SEQUENCES[algo]:
        for i in fz.steps(kind, nb):
            received = {r: set() for r in range(world)}
            for phase in fz.plan_step(kind, i, nb, world):
                for op in phase.ops:
                    have = held[op.rank] | received[op.rank]
                    missing = [k for k in op.ins if k not in have]
                    assert not missing, (kind, i, op, missing)
                    held[op.rank].update(op.outs)
                seen = set()
                for src, dst, key in phase.sends:
                    assert src != dst
                    assert (key, dst) not in seen, (kind, i, key, dst)
                    seen.add((key, dst))
                    assert key in held[src] | received[src], (kind, i, key, src)
                    assert key not in held[dst] and key not in received[dst], (kind, i, key, dst)
                    received[dst].add(key)
                    total_sends += 1
    return held, total_sends


@pytest.mark.parametrize("algo", sorted(SEQUENCES))
@pytest.mark.parametrize("world", range(1, 9))
def test_plan_inputs_are_held_and_sends_are_needed(algo, world):
    for nb in range(1, 21):
        held, sends = _simulate(algo, nb, world)
        if world == 1:
            assert sends == 0
        # every result block ends on its owner
        name = "X" if algo == "inverse" else "A"
        for r in range(nb):
            for c in range(nb):
                if algo != "cholesky" or r >= c:
                    assert (name, r, c) in held[comm.elem_owner(r, c, nb, world)]


@pytest.mark.parametrize("kind", fz.KINDS)
def test_plan_is_a_pure_function(kind):
    for nb in (1, 2, 7, 13):
        for world in (1, 3, 8):
            for i in fz.steps(kind, nb):
                a = fz.plan_step(kind, i, nb, world)
                b = fz.plan_step(kind, i, nb, world)
                assert a == b
                # the same list whichever rank asks: the plan takes no rank
                assert all(isinstance(p, fz.Phase) for p in a)


def test_plan_one_rank_sends_nothing():
    for kind in fz.KINDS:
        for nb in range(1, 21):
            for i in fz.steps(kind, nb):
                assert all(not p.sends for p in fz.plan_step(kind, i, nb, 1))


def test_grid_matches_the_block_row_split():
    """The factorization grid is the one toBlockMatrix(nb, nb) would build: same block length, no empty block."""
    for n in range(1, 400):
        for base in (1, 2, 3, 7, 40, 128, 1000):
            nb, sub = fz.grid(n, base)
            assert sub * (nb - 1) < n <= sub * nb

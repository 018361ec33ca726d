"""The PageRank example on the GPU: ranks bit for bit against the sparse oracle (small graphs, an R-MAT scale-20 graph, a
star, rows at each bin bound) and the dense reference model; against the dense composition of this repository's own
public operations within an fp64 bound, with the same errors where that composition raises; mb_pagerank_train against
a loop of mb_pagerank_step; the C ABI's errors; two ranks against one; and the example's main on a link file."""
import os
import socket
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from tests import pagerank_oracle as po

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]


def _matrix(src, dst, n):
    import marlin_b200 as mb
    return mb.SparseVecMatrix(po.link_rows(src, dst, n), n, n)


def _pieces(dv):
    return [v.toBreeze().reshape(-1) for _, v in sorted(dv.vectors, key=lambda t: t[0])]


def _assert_bits(got, want):
    assert [len(g) for g in got] == [len(w) for w in want]
    for g, w in zip(got, want):
        assert np.array_equal(g.view(np.int64), w.view(np.int64))


def _dense_rows(ids, rowptr, cols, vals, n):
    out = {}
    for r, page in enumerate(ids):
        v = np.zeros(n)
        v[cols[rowptr[r]:rowptr[r + 1]]] = vals[rowptr[r]:rowptr[r + 1]]
        out[int(page)] = v
    return out


@pytest.mark.parametrize("n", [4, 5, 7, 64, 257, 1000])
def test_small_graphs_match_the_sparse_oracle_and_the_dense_reference(n):
    from marlin_b200.examples import page_rank as pr
    src, dst = po.random_graph(n, seed=1000 + n)
    rows = po.link_rows(src, dst, n)
    m = _matrix(src, dst, n)
    for iterations in (1, 3, 20):
        got = _pieces(pr.pageRank(m, iterations))
        _assert_bits(got, po.InLinks(*rows, n).run(iterations))
        _assert_bits(got, po.dense(_dense_rows(*rows, n), n, iterations))


def test_rmat_scale_20():
    from marlin_b200.examples import page_rank as pr
    n = 1 << 20
    src, dst = po.rmat(20, 16, seed=5)
    rows = po.link_rows(src, dst, n)
    import marlin_b200 as mb
    got = _pieces(pr.pageRank(mb.SparseVecMatrix(rows, n, n), 10))
    _assert_bits(got, po.InLinks(*rows, n).run(10))


def test_star():
    """One page with 2^20 - 1 in-links: one warp's serial chain over both segments."""
    from marlin_b200.examples import page_rank as pr
    n = 1 << 20
    src = np.concatenate([np.arange(1, n), [0]])
    dst = np.concatenate([np.zeros(n - 1, np.int64), [n - 1]])
    got = _pieces(pr.pageRank(_matrix(src, dst, n), 3))
    _assert_bits(got, po.InLinks(*po.link_rows(src, dst, n), n).run(3))


def test_rows_at_each_bin_bound():
    """In-degrees on both sides of MB_PAGERANK_LIGHT_BOUND, heavy rows inside warps of light rows (so a warp's light rows
    form several runs), runs whose edges span several stages, empty rows, and in-links on both sides of the segment
    boundary."""
    from marlin_b200 import _native as nat
    from marlin_b200.examples import page_rank as pr
    b = nat.MB_PAGERANK_LIGHT_BOUND
    rng = np.random.default_rng(3)
    n = 8192
    pattern = [0, 1, 2, 31, 32, b - 1, b, b + 1, b + 2, 2 * b, 700, 5000, 0, 1]
    deg = np.array([pattern[t % len(pattern)] if t % 3 else 200 for t in range(n)])
    deg[64:96] = b                                         # one warp of rows exactly at the bound
    deg[96:128] = b + 1                                    # one warp of rows just above it
    src = np.concatenate([rng.choice(n, d, replace=False) for d in deg])
    dst = np.repeat(np.arange(n), deg)
    rows = po.link_rows(src, dst, n)
    got = _pieces(pr.pageRank(_matrix(src, dst, n), 4))
    _assert_bits(got, po.InLinks(*rows, n).run(4))


def _c_links(n, src, dst):
    from marlin_b200.examples import page_rank as pr
    rows = po.link_rows(src, dst, n)
    return pr._in_links([rows], n, 0, n)


def _vec(t):
    from marlin_b200.matrix.sub_matrix import SubMatrix
    return SubMatrix(buf=t, rows=t.numel(), cols=1, ld=max(1, t.numel()))


def test_train_is_a_loop_of_steps():
    import torch
    from marlin_b200 import _native as nat
    from marlin_b200.runtime import Runtime
    rt = Runtime.get()
    n = 5000
    src, dst = po.rmat(12, 8, seed=9)
    src, dst = src % n, dst % n
    L = _c_links(n, src, dst)
    seg = (n + 1) // 2
    x = torch.rand(n, dtype=torch.float64, device=rt.device)
    a, b = x.clone(), torch.empty_like(x)
    rt.sync_stream()
    for _ in range(7):
        av, bv = _vec(a), _vec(b)                          # held: their handles must outlive the call
        nat.check(rt.lib.mb_pagerank_step(rt.ctx, L.handle(), av.handle(), seg, 0.15, bv.handle()))
        a, b = b, a
    t = x.clone()
    tv = _vec(t)
    nat.check(rt.lib.mb_pagerank_train(rt.ctx, L.handle(), seg, 0.15, 7, tv.handle()))
    assert torch.equal(t.view(torch.int64), a.view(torch.int64))
    z = x.clone()
    zv = _vec(z)
    nat.check(rt.lib.mb_pagerank_train(rt.ctx, L.handle(), seg, 0.15, 0, zv.handle()))
    assert torch.equal(z, x)


def test_iterations_zero_gives_ones():
    from marlin_b200.examples import page_rank as pr
    for n in (1, 2, 5, 1000):
        got = _pieces(pr.pageRank(_matrix([0], [n - 1], n), 0))
        s = (n + 1) // 2
        _assert_bits(got, [np.ones(s), np.ones(n - s)])


def test_c_abi_errors():
    import torch
    from marlin_b200 import _native as nat
    from marlin_b200.runtime import Runtime
    rt = Runtime.get()
    n = 100
    L = _c_links(n, np.arange(n), (np.arange(n) * 7) % n)
    x = torch.ones(n, dtype=torch.float64, device=rt.device)
    y = torch.empty(n, dtype=torch.float64, device=rt.device)
    short = torch.empty(n - 1, dtype=torch.float64, device=rt.device)
    rt.sync_stream()

    def step(xt, seg, yt):
        xv, yv = _vec(xt), _vec(yt)                        # held: their handles must outlive the call
        nat.check(rt.lib.mb_pagerank_step(rt.ctx, L.handle(), xv.handle(), seg, 0.15, yv.handle()))

    for seg in (0, -5):
        with pytest.raises(nat.MarlinArgumentError, match="segment length") as e:
            step(x, seg, y)
        assert e.value.code == nat.MB_ERR_INVALID_ARG
    for xv, yv in ((short, y), (x, short)):
        with pytest.raises(nat.MarlinArgumentError, match="expected") as e:
            step(xv, 50, yv)
        assert e.value.code == nat.MB_ERR_DIM_MISMATCH
    with pytest.raises(nat.MarlinArgumentError, match="overlaps"):
        step(x, 50, x)
    from marlin_b200.examples import page_rank as pr
    half = pr._in_links([po.link_rows(np.arange(n), np.arange(n), n)], n, 0, 50)
    with pytest.raises(nat.MarlinArgumentError, match="square") as e:
        xv = _vec(x)
        nat.check(rt.lib.mb_pagerank_train(rt.ctx, half.handle(), 50, 0.15, 1, xv.handle()))
    assert e.value.code == nat.MB_ERR_DIM_MISMATCH
    step(x, 50, y)                                        # still usable after the errors
    rt.synchronize()


def _composition(m, n, iterations):
    """The example written with this repository's own public dense operations."""
    import marlin_b200 as mb
    links = m.toDenseVecMatrix().transpose(2).multiply(0.85)
    ranks = mb.MTUtils.onesDistVector(None, n, 2)
    for _ in range(iterations):
        res = links.multiply(ranks)
        acc = None
        for _, v in sorted(res.getVectors, key=lambda t: t[0]):
            acc = v.toBreeze().reshape(-1) if acc is None else acc + v.toBreeze().reshape(-1)
        ranks = mb.DistributedVector.fromVector(None, acc + np.ones(n) * 0.15, 2)
    return _pieces(ranks)


@pytest.mark.parametrize("n", [4, 9, 300])
def test_dense_composition_within_fp64_bound(n):
    """The existing gemv folds its column chunks, so the composition is not F2J-exact: each step may differ by the
    rounding of a reordered sum of at most n non-negative terms, n * u * y per element, over `iterations` steps (the
    damping 0.85 < 1 keeps earlier differences from growing)."""
    from marlin_b200.examples import page_rank as pr
    src, dst = po.random_graph(n, seed=n)
    m = _matrix(src, dst, n)
    iterations = 6
    got = np.concatenate(_pieces(pr.pageRank(m, iterations)))
    want = np.concatenate(_composition(m, n, iterations))
    u = np.finfo(np.float64).eps / 2
    assert np.all(np.abs(got - want) <= 2 * iterations * n * u * np.abs(want))


@pytest.mark.parametrize("n", [1, 2, 3])
def test_small_graphs_raise_as_the_dense_composition(n):
    from marlin_b200.examples import page_rank as pr
    m = _matrix([0], [n - 1], n)
    with pytest.raises(Exception) as want:
        _composition(m, n, 1)
    with pytest.raises(type(want.value)) as got:
        pr.pageRank(m, 1)
    assert str(got.value) == str(want.value)


def test_two_ranks_bit_identical_to_one(tmp_path):
    import marlin_b200 as mb
    from marlin_b200.examples import page_rank as pr
    sys.path.insert(0, str(ROOT / "tests"))
    import pagerank_gpu_worker as w
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    env = dict(os.environ, PAGERANK_WORKER_OUT=str(tmp_path / "r"))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), str(ROOT / "tests" / "pagerank_gpu_worker.py")]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900, env=env)
    assert out.returncode == 0, out.stdout[-4000:]
    for r in range(2):
        assert f"rank {r} small graph raised" in out.stdout and f"rank {r} pagerank ok" in out.stdout
    src, dst = w.data()
    one = _pieces(pr.pageRank(mb.SparseVecMatrix(po.link_rows(src, dst, w.N), w.N, w.N), w.ITERATIONS))
    two = [np.load(str(tmp_path / f"r.{r}.npz"))[f"p{r}"] for r in range(2)]       # piece i on rank i
    _assert_bits(two, one)


def test_main_prints_the_oracle_ranks():
    """tests/golden/pagerank.links is a hand-written link file (`source target` per line, pages 1-based, the input of
    examples/PageRank.scala): 8 pages with a duplicated line, a self-link, a tab and an extra token, a blank line, and
    page 8 with neither out-links nor in-links."""
    from marlin_b200.utils.mt_utils import _jdouble
    path = ROOT / "tests" / "golden" / "pagerank.links"
    out = subprocess.run([sys.executable, "-m", "marlin_b200.examples.page_rank", str(path), "5", "8"], cwd=str(ROOT),
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-3000:]
    lines = [l for l in path.read_text().splitlines() if l.strip()]
    want = po.dense(po.literal_rows(lines, 8), 8, 5)
    got = [l for l in out.stdout.splitlines() if l.startswith("ranks: ")]
    assert got == ["ranks: " + ", ".join(_jdouble(v) for v in p) for p in want]
    assert [l for l in out.stdout.splitlines() if l.startswith("in iteration")] == [f"in iteration {i}" for i in range(5)]
    assert sum(l.startswith("index: ") for l in out.stdout.splitlines()) == 7          # page 8 has no out-links

"""The matrix-file writer on the H100 (mb_save_rows, mb_save_blocks and the Python save methods on top of them): the files
equal the oracle's line restatements (oracle/reference_model.py save_lines / save_block_lines, whose tokens are
mt_utils._jdouble) byte for byte, and the device tokens equal the host build of the same core (tests/test_text_host.py)."""
import ctypes as C
import os
import socket
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from marlin_b200 import _native as nat
from marlin_b200.utils.mt_utils import _jdouble
from tests.test_gpu_temporaries import _Pool
from tests.test_text_host import build_text_driver, tokens

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
CHUNK = nat.MB_TEXT_CHUNK_VALUES


@pytest.fixture(scope="module")
def M():
    import marlin_b200 as mb
    mb.Runtime.get()
    return mb


def rt(M):
    r = M.Runtime.get()
    r.sync_stream()
    return r


def chunks(n):
    return -(-n // CHUNK)


def save_blocks(M, blocks, path):
    """mb_save_blocks over [((r, c), SubMatrix)]; returns the launches it made."""
    r = rt(M)
    handles = (nat.c_blk * max(1, len(blocks)))(*[s.handle() for _, s in blocks])
    rc = np.array([list(k) for k, _ in blocks], dtype=np.int32).reshape(-1)
    l0 = r.launch_count()
    nat.check(r.lib.mb_save_blocks(r.ctx, handles, rc.ctypes.data_as(C.c_void_p), len(blocks), os.fsencode(str(path))))
    return r.launch_count() - l0


def block_line(r, c, arr):
    return f"{r}-{c}-{arr.shape[0]}-{arr.shape[1]}:" + ",".join(_jdouble(v) for v in arr.reshape(-1, order="F")) + "\n"


def test_random_bit_patterns_match_the_host_core(M, tmp_path):
    """One 1 x 2^24 line of random bit patterns: eight chunks, so the line crosses chunk boundaries seven times."""
    n = 1 << 24
    bits = np.random.default_rng(7).integers(0, 2 ** 64, size=n, dtype=np.uint64)
    buf = torch.from_numpy(bits.view(np.float64).copy()).to(M.Runtime.get().device)
    blk = M.SubMatrix(buf=buf, rows=1, cols=n, ld=1)
    launches = save_blocks(M, [((3, 4), blk)], tmp_path / "part")
    assert launches == 2 * chunks(n) and chunks(n) == 8
    text = (tmp_path / "part").read_text()
    head = f"3-4-1-{n}:"
    assert text.startswith(head) and text.endswith("\n") and text.count("\n") == 1
    got = text[len(head):-1].split(",")
    assert len(got) == n
    want = tokens(bits.tolist(), build_text_driver())
    assert got == want
    pick = np.random.default_rng(8).choice(n, size=1_000_000, replace=False)
    vals = bits[pick].view(np.float64)
    assert [got[i] for i in pick.tolist()] == [_jdouble(v) for v in vals.tolist()]


SPECIAL = np.array([0.0, -0.0, np.nan, -np.nan, np.inf, -np.inf, 5e-324, -5e-324, 2.225073858507201e-308,
                    1.7976931348623157e308, 9.999999999999998e-4, 0.001, 9999999.999999998, 1e7, 2.0 ** 53 + 2, 0.1, -1.5])


def row_cases():
    rng = np.random.default_rng(11)
    nan_payload = np.array([0x7FF0000000000123, 0xFFF8000000000001], dtype=np.uint64).view(np.float64)
    return {
        "random": (np.arange(300), rng.random((300, 77)) * 10.0 ** rng.integers(-12, 12, (300, 77))),
        "special": (np.arange(6), np.resize(np.concatenate([SPECIAL, nan_payload]), (6, 19))),
        "ids_to_2_40": (np.array([2 ** 40, 5, 2 ** 40 - 1, 0, 123456789012]), rng.standard_normal((5, 9))),
        "one_by_one": (np.array([0]), np.array([[0.3]])),
        "zero_columns": (np.array([4, 1, 2 ** 33]), np.zeros((3, 0))),
        "one_column": (np.arange(2000), rng.random((2000, 1))),
    }


@pytest.mark.parametrize("case", list(row_cases()))
def test_rows_equal_save_lines(M, oracle, tmp_path, case):
    ids, arr = row_cases()[case]
    m = M.DenseVecMatrix(list(zip(ids.tolist(), arr)))
    r = rt(M)
    l0 = r.launch_count()
    m.saveWithDescription(str(tmp_path / "out"))
    assert r.launch_count() - l0 == 2 * chunks(arr.size)
    om = oracle.DenseVecMatrix(list(zip(ids.tolist(), arr)))
    assert (tmp_path / "out" / "part-00000").read_text() == "".join(x + "\n" for x in om.save_lines())
    assert (tmp_path / "out" / "_description").read_text() == om.description()


def test_empty_shard_writes_an_empty_file(M, tmp_path):
    M.DenseVecMatrix([], nRows=4, nCols=3).saveToFileSystem(str(tmp_path / "out"))
    assert (tmp_path / "out" / "part-00000").read_bytes() == b""


def test_sliced_and_transposed_views(M, oracle, tmp_path):
    rng = np.random.default_rng(12)
    big = M.SubMatrix(rng.standard_normal((90, 70)))                        # column-major
    view = big.slice(7, 60, 3, 66)
    want = view.toBreeze()
    ids = np.arange(100, 100 + want.shape[0])
    # a column-major view as a row shard: read row by row through the strides, no copy
    M.DenseVecMatrix(ids=ids, data=view, nRows=200, nCols=want.shape[1]).saveToFileSystem(str(tmp_path / "rows"))
    om = oracle.DenseVecMatrix(list(zip(ids.tolist(), want)))
    assert (tmp_path / "rows" / "part-00000").read_text() == "".join(x + "\n" for x in om.save_lines())
    # blocks: a slice, a transposed view and a transposed slice
    pieces = [((0, 0), view), ((0, 1), big.t), ((1, 0), big.t.slice(5, 40, 11, 12))]
    save_blocks(M, pieces, tmp_path / "blocks")
    assert (tmp_path / "blocks").read_text() == "".join(block_line(r, c, s.toBreeze()) for (r, c), s in pieces)


def test_block_matrix_save_to_file_system(M, oracle, tmp_path):
    rng = np.random.default_rng(13)
    rows = [(i, rng.random(33) * 1e-5) for i in range(41)]
    bm = M.DenseVecMatrix(rows).toBlockMatrix(3, 2)
    bm.saveToFileSystem(str(tmp_path / "b"), "BlockMatrix")
    want = oracle.DenseVecMatrix(rows).to_block_matrix(3, 2).save_block_lines()
    got = (tmp_path / "b" / "part-00000").read_text()
    assert sorted(got.splitlines(keepends=True)) == sorted(x + "\n" for x in want)


def test_float32_and_empty_blocks_and_long_block(M, tmp_path):
    """fp32 widens exactly; a block without values is its header alone; a block of more than MB_TEXT_CHUNK_VALUES."""
    dev = M.Runtime.get().device
    rng = np.random.default_rng(14)
    f32 = np.concatenate([rng.standard_normal(997).astype(np.float32), np.array([np.nan, np.inf, 1e-45, 3.4e38, -0.0], np.float32)])
    fblk = M.SubMatrix(buf=torch.from_numpy(f32).to(dev), rows=6, cols=167, ld=6)
    n = CHUNK + 4099
    big = rng.standard_normal(n)
    bblk = M.SubMatrix(buf=torch.from_numpy(big).to(dev), rows=CHUNK // 16 + 1, cols=16, ld=CHUNK // 16 + 1)
    n = bblk.rows * bblk.cols
    empty = M.SubMatrix(buf=torch.empty(0, dtype=torch.float64, device=dev), rows=0, cols=4, ld=1)
    blocks = [((0, 0), fblk), ((7, 2 ** 30), empty), ((1, 1), bblk)]
    launches = save_blocks(M, blocks, tmp_path / "part")
    assert launches == 2 * (chunks(fblk.rows * fblk.cols) + chunks(n)) and chunks(n) == 2
    text = (tmp_path / "part").read_text()
    want = (block_line(0, 0, f32[: 6 * 167].astype(np.float64).reshape((6, 167), order="F")) + f"7-{2 ** 30}-0-4:\n"
            + block_line(1, 1, big[:n].reshape((bblk.rows, 16), order="F")))
    assert text == want


def test_unwritable_path_is_an_io_error_and_frees_everything(M, tmp_path):
    pool = _Pool()
    r = rt(M)
    m = M.DenseVecMatrix([(i, np.arange(5.0) + i) for i in range(10)])
    (tmp_path / "bad" / "part-00000").mkdir(parents=True)
    torch.cuda.synchronize()
    before = pool.used()
    with pytest.raises(nat.MarlinError) as ei:
        m.saveToFileSystem(str(tmp_path / "bad"))
    assert ei.value.code == nat.MB_ERR_IO and "part-00000" in ei.value.message
    blk = M.SubMatrix(np.ones((3, 3)))
    with pytest.raises(nat.MarlinError) as ei:
        save_blocks(M, [((0, 0), blk)], tmp_path / "bad" / "part-00000")
    assert ei.value.code == nat.MB_ERR_IO
    r.synchronize()
    torch.cuda.synchronize()
    assert pool.used() == before


def test_two_ranks_write_their_own_parts(M, oracle, tmp_path):
    sys.path.insert(0, str(ROOT / "tests"))
    import text_gpu_worker as w
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    env = dict(os.environ, TEXT_WORKER_OUT=str(tmp_path / "out"))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), str(ROOT / "tests" / "text_gpu_worker.py")]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900, env=env)
    assert out.returncode == 0, out.stdout[-4000:]
    parts = [(tmp_path / "out" / f"part-{r:05d}").read_text() for r in range(2)]
    for r in range(2):
        assert parts[r] == "".join(x + "\n" for x in oracle.DenseVecMatrix(w.rows(r)).save_lines())
    both = oracle.DenseVecMatrix(w.rows(0) + w.rows(1)).save_lines()
    assert (parts[0] + parts[1]).splitlines() == both

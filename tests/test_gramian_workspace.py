"""Temporary device memory of the Gramian (mb_gramian_workspace_bytes, pure host logic): K is split only when the lower
triangle of 128 x 128 tiles is too small for the SMs, and the split-K partials never take more than 256 MiB, so every
column count the 65535 cap allows needs no more memory than G itself."""
import pytest

from marlin_b200 import _native as nat

CAP = 256 << 20


@pytest.fixture(scope="module")
def lib():
    return nat.load()


def test_workspace_is_bounded_for_every_size(lib):
    for sms in (1, 8, 114, 132, 264):
        for n in list(range(1, 3000, 37)) + [4096, 8192, 16384, 20000, 32768, 40000, 65535]:
            for m in (1, 511, 4096, 1 << 17, 1 << 20, (1 << 31) - 1):
                b = lib.mb_gramian_workspace_bytes(n, m, sms)
                assert 0 <= b <= CAP, (n, m, sms, b)
                t = (n + 127) // 128
                if t * (t + 1) // 2 >= 2 * sms:
                    assert b == 0, (n, m, sms, b)             # enough tiles: no split, the product goes into G
                ldw = (n + 1) & ~1
                assert b % (8 * ldw * n) == 0


def test_split_k_is_used_where_the_triangle_is_small(lib):
    # n = 1024 on 132 SMs: 36 tiles; 11 splits fill three waves exactly (88 MiB of partials)
    assert lib.mb_gramian_workspace_bytes(1024, 1 << 20, 132) == 11 * 1024 * 1024 * 8
    # too few rows to split (>= 512 rows per split), and a single tile row never splits past the cap
    assert lib.mb_gramian_workspace_bytes(1024, 600, 132) == 0
    assert lib.mb_gramian_workspace_bytes(2816, 1 << 20, 132) <= CAP
    assert lib.mb_gramian_workspace_bytes(65535, 1 << 20, 132) == 0
    assert lib.mb_gramian_workspace_bytes(0, 1 << 20, 132) == 0

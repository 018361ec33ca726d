"""The formatter core of the matrix-file writer (marlin_b200/csrc/text.h) built as plain host C++ with g++, against the
Double.toString restatement it must match byte for byte (mt_utils._jdouble), and its generated 5^q tables against
Python integers.  No GPU needed."""
import re
import shutil
import struct
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from marlin_b200.utils.mt_utils import _jdouble

ROOT = Path(__file__).resolve().parents[1]
CSRC = ROOT / "marlin_b200" / "csrc"
BIN = ROOT / "scripts" / "bin"


def build_text_driver() -> Path:
    """tests/cpp/text_driver.cpp (the core and a stdin/stdout loop) with g++ -Werror into scripts/bin/text_driver."""
    exe = BIN / "text_driver"
    BIN.mkdir(parents=True, exist_ok=True)
    cmd = [shutil.which("g++") or "g++", "-std=c++17", "-O2", "-Wall", "-Wextra", "-Werror", f"-I{CSRC}",
           str(ROOT / "tests" / "cpp" / "text_driver.cpp"), "-o", str(exe)]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert out.returncode == 0, out.stdout
    return exe


def tokens(bits, exe=None) -> list:
    """The core's token of every 64-bit pattern in bits."""
    exe = exe or build_text_driver()
    out = subprocess.run([str(exe), "d"], input="".join(f"{int(b):016x}\n" for b in bits), stdout=subprocess.PIPE,
                         stderr=subprocess.PIPE, text=True, timeout=600)
    assert out.returncode == 0, out.stderr
    got = out.stdout.split("\n")
    assert got[-1] == ""
    return got[:-1]


def f2b(v: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", v))[0]


def b2f(b: int) -> float:
    return struct.unpack("<d", struct.pack("<Q", b))[0]


def neighbours(b: int):
    return [x for x in (b - 1, b, b + 1) if 0 <= x < 1 << 64]


@pytest.fixture(scope="module")
def exe():
    return build_text_driver()


def check(exe, bits):
    bits = [int(b) & (2 ** 64 - 1) for b in bits]
    got = tokens(bits, exe)
    assert len(got) == len(bits)
    bad = [(f"{b:016x}", g, _jdouble(b2f(b))) for b, g in zip(bits, got) if g != _jdouble(b2f(b))]
    assert not bad, bad[:10]
    return got


def test_special_values(exe):
    nans = [0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0xFFF0000000000001, 0x7FFFFFFFFFFFFFFF,
            0xFFFFFFFFFFFFFFFF, 0x7FF4000000000000]
    got = check(exe, nans + [0x7FF0000000000000, 0xFFF0000000000000, 0, 1 << 63])
    assert got == ["NaN"] * len(nans) + ["Infinity", "-Infinity", "0.0", "-0.0"]


def test_range_ends(exe):
    got = check(exe, [1, 0x000FFFFFFFFFFFFF, 0x0010000000000000, 0x7FEFFFFFFFFFFFFF])
    assert got == ["5.0E-324", "2.225073858507201E-308", "2.2250738585072014E-308", "1.7976931348623157E308"]
    check(exe, [b | 1 << 63 for b in (1, 0x000FFFFFFFFFFFFF, 0x0010000000000000, 0x7FEFFFFFFFFFFFFF)])


def test_min_value_keeps_the_shortest_digit(exe):
    """Double.MIN_VALUE: _jdouble and the core print the one shortest digit, 5.0E-324, where JDK 19+ prints the closer
    4.9E-324.  Both change together or not at all."""
    assert _jdouble(5e-324) == "5.0E-324"
    assert tokens([1], exe) == ["5.0E-324"]


def test_every_power_of_two_and_its_neighbours(exe):
    check(exe, [n for e in range(-1074, 1024) for n in neighbours(f2b(2.0 ** e))])


def test_every_power_of_ten_and_its_neighbours(exe):
    bits = []
    for e in range(-324, 309):
        v = float(f"1e{e}")
        if v != 0.0 and v != float("inf"):
            bits += neighbours(f2b(v))
    assert len(bits) > 1800
    check(exe, bits)


def test_notation_boundaries(exe):
    got = check(exe, [f2b(v) for v in (9.999999999999998e-4, 0.001, 9999999.999999998, 1.0e7)])
    assert got == ["9.999999999999998E-4", "0.001", "9999999.999999998", "1.0E7"]
    check(exe, neighbours(f2b(0.001)) + neighbours(f2b(1e7)) + [f2b(-v) for v in (0.001, 1e7, 123.0, 1e6, 0.0123)])


def test_integers_near_2_53(exe):
    base = 2 ** 53
    check(exe, [f2b(float(base + k)) for k in range(-40, 41)] + [f2b(-float(base + k)) for k in range(-40, 41, 3)])


def test_random_bit_patterns(exe):
    rng = np.random.default_rng(20261018)
    check(exe, rng.integers(0, 2 ** 64, size=200_000, dtype=np.uint64, endpoint=False).tolist())


def test_uniform_values(exe):
    rng = np.random.default_rng(20261019)
    check(exe, rng.random(200_000).view(np.uint64).tolist())


def test_long_tokens(exe):
    vals = [0, 1, -1, -2 ** 63, 2 ** 63 - 1, 10, -10, 99, 2 ** 40, -(2 ** 31)]
    out = subprocess.run([str(exe), "l"], input="".join(f"{v}\n" for v in vals), stdout=subprocess.PIPE, text=True, timeout=60)
    assert out.returncode == 0
    assert out.stdout.split("\n")[:-1] == [str(v) for v in vals]


def test_generated_tables_match_python_integers():
    """text_tables.h is what scripts/gen_text_tables.py writes, and every entry is the integer its comment defines."""
    sys.path.insert(0, str(ROOT / "scripts"))
    import gen_text_tables as g
    header = (CSRC / "text_tables.h").read_text()
    assert g.header() == header
    def table(name):
        body = header.split(f"#define {name} {{", 1)[1].split("}", 1)[0]
        w = [int(x, 16) for x in re.findall(r"0x([0-9a-f]{16})ull", body)]
        return [lo | hi << 64 for lo, hi in zip(w[0::2], w[1::2])]
    pow5, inv = table("MB_TEXT_POW5_TABLE"), table("MB_TEXT_POW5_INV_TABLE")
    assert len(pow5) == 326 and len(inv) == 291
    for i, v in enumerate(pow5):
        p = 5 ** i
        assert v.bit_length() == 125 and v == (p >> (p.bit_length() - 125) if p.bit_length() >= 125 else p << (125 - p.bit_length()))
    for q, v in enumerate(inv):
        p = 5 ** q
        assert v == (1 << (p.bit_length() - 1 + 125)) // p + 1

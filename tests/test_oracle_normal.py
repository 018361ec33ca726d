"""The StandardNormalGenerator oracle (tests/normal_oracle.py) without a GPU: the vectorised stream against the scalar
nextGaussian restatement, the vectorised log against both existing fdlibm restatements (tests/als_oracle.py and
marlin_b200/csrc/hostlogic.cpp), and the distribution of the values."""
import ctypes as C
import re
import shutil
import struct
import subprocess
from pathlib import Path

import numpy as np
import pytest
import scipy.stats

from tests import als_oracle as ao
from tests import normal_oracle as no

ROOT = Path(__file__).resolve().parents[1]


@pytest.fixture(scope="module")
def cpp_log(tmp_path_factory):
    """hostlogic.cpp's fdlibm_log, compiled on its own (it sits in an anonymous namespace of that translation unit)."""
    d = tmp_path_factory.mktemp("fdlibm")
    src = d / "log.cpp"
    src.write_text(f'#include "{ROOT / "marlin_b200" / "csrc" / "hostlogic.cpp"}"\n'
                   'int32_t mb_fail(int32_t code, const char*, ...) { return code; }\n'      # the library's error sink
                   'extern "C" double restated_fdlibm_log(double x) { return fdlibm_log(x); }\n')
    lib = d / "liblog.so"
    out = subprocess.run([shutil.which("g++") or "g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC",
                          str(src), "-o", str(lib)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert out.returncode == 0, out.stdout
    so = C.CDLL(str(lib))
    so.restated_fdlibm_log.restype = C.c_double
    so.restated_fdlibm_log.argtypes = [C.c_double]
    return so.restated_fdlibm_log


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


@pytest.mark.parametrize("seed", [0, -1, 42, 123456789, -(2 ** 63), 2 ** 63 - 1])
def test_vectorised_stream_equals_scalar_next_gaussian(oracle, seed):
    n = 2001                                               # odd: the last pair's second value is dropped
    vals, positions, _ = no.normal_stream(seed, n, chunk=1 << 10)
    rnd = no.XORShiftNormal(seed)
    ref = np.array([rnd.next_value() for _ in range(n)])
    assert np.array_equal(_bits(vals), _bits(ref))
    # the scalar generator has drawn exactly 2A nextDoubles (next(26) and next(27) each), and holds the dropped value
    probe = no.XORShiftNormal(seed)
    for _ in range(n):
        probe.next_value()
    assert probe.have_next
    steps = 0
    state = no.XORShiftNormal(seed).seed
    while state != probe.seed:
        state = _step(state)
        steps += 1
        assert steps <= 2 * positions
    assert steps == 2 * positions                          # two XORShift steps per nextDouble


def _step(s):
    s ^= (s << 21) & no.M64
    s ^= s >> 35
    s ^= (s << 4) & no.M64
    return s


@pytest.mark.parametrize("mean,variance", [(3.5, 0.25), (-1e300, 4.0), (-0.0, 0.0), (1.0, -1.0), (0.0, float("nan"))])
def test_vectorised_scaling_equals_scalar(oracle, mean, variance):
    vals, _, _ = no.normal_stream(7, 301, mean, variance, chunk=1 << 10)
    rnd = no.XORShiftNormal(7, mean, variance)
    ref = np.array([rnd.next_value() for _ in range(301)])
    if variance < 0 or variance != variance:
        assert np.isnan(vals).all() and np.isnan(ref).all()
    else:
        assert np.array_equal(_bits(vals), _bits(ref))
    if variance == 0.0:
        assert {struct.pack("<d", v) for v in vals} <= {struct.pack("<d", 0.0), struct.pack("<d", -0.0)}
        assert (np.signbit(vals)).any() and (~np.signbit(vals)).any()      # -0.0 + (+0.0) and -0.0 + (-0.0)


def _log_edges():
    rng = np.random.default_rng(5)
    xs = [rng.uniform(0, 1, 4000), rng.uniform(0, 1, 1000) ** 8]
    xs.append(np.array([2.0 ** -e for e in range(1, 1023)]))                            # powers of two: f == 0
    ulp_near_1 = np.nextafter(1.0, 0.0)
    xs.append(np.array([1.0 - d for d in np.linspace(2.0 ** -53, 2.0 ** -20, 600)] + [ulp_near_1]))     # within 2^-20 of 1
    xs.append(np.array([2.0 ** -e * (1 + d) for e in range(1, 60) for d in (2.0 ** -21, 2.0 ** -20, 3 * 2.0 ** -22)]))
    # around the i > 0 split: hx = 0x6147a .. 0x6b851 (high-word significand bits), at both ends and for k == 0 and not
    edges = []
    for hx in (0x6147A - 1, 0x6147A, 0x6147A + 1, 0x6B851 - 1, 0x6B851, 0x6B851 + 1, 0x6A09E, 0x6A09F, 0x95F63 ^ 0xFFFFF):
        for exp in (0x3FE, 0x3FD, 0x3F0, 0x100):
            for lo in (0, 1, 0xFFFFFFFF):
                edges.append(struct.unpack("<d", struct.pack("<Q", ((exp << 20 | (hx & 0xFFFFF)) << 32) | lo))[0])
    xs.append(np.array([x for x in edges if 0 < x < 1]))
    xs.append(np.array([2.0 ** -1022, 2.0 ** -1022 * 1.5, 0.5, 0.75, 0.7071067811865476, 0.7071067811865475]))
    return np.concatenate(xs)


def test_vectorised_log_equals_both_restatements(cpp_log):
    x = _log_edges()
    x = x[(x > 0) & (x < 1)]
    counts = {}
    got = no.fdlibm_log_vec(x, counts)
    py = np.array([ao.fdlibm_log(float(v)) for v in x])
    cc = np.array([cpp_log(float(v)) for v in x])
    assert np.array_equal(_bits(got), _bits(py))
    assert np.array_equal(_bits(got), _bits(cc))
    assert all(counts[b] > 0 for b in no.BRANCHES), counts
    # it is a log: within 1 ulp of numpy's
    assert np.all(np.abs(got - np.log(x)) <= np.spacing(np.abs(np.log(x))))


def test_values_are_normally_distributed(oracle):
    mean, variance = 3.5, 0.25
    vals, positions, counts = no.normal_stream(2024, 10 ** 6, mean, variance)
    assert positions >= 10 ** 6                            # 2A >= n: at least one nextDouble per value
    z = (vals - mean) / 0.5
    ks = scipy.stats.kstest(z, "norm")
    assert ks.pvalue > 1e-3, ks
    assert abs(z.mean()) < 5 / 1000                      # 5 standard errors of 10^6 draws
    assert abs(z.var() - 1) < 5 * np.sqrt(2) / 1000
    assert abs(scipy.stats.skew(z)) < 5 * np.sqrt(6) / 1000
    assert abs(scipy.stats.kurtosis(z)) < 5 * np.sqrt(24) / 1000
    # acceptance of the polar method: pi / 4
    assert abs(10 ** 6 / positions - np.pi / 4) < 0.01


def test_documented_tile_size_is_the_one_the_tests_use():
    header = (ROOT / "include" / "marlin_b200.h").read_text()
    assert int(re.search(r"#define MB_NORMAL_TILE_ATTEMPTS (\d+)", header).group(1)) == 32768

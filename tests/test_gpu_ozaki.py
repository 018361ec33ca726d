"""fp64 GEMM on the int8 tensor cores (wgmma .s32.s8.s8, Ozaki digit-plane split) — opt-in mode of the C ABI.

Checked against the fp64 oracle on the same inputs with the tolerance BASELINE.json states for fp64 (1e-10):
    max_ij |C - C_ref| / (rowmax_i(|A|) * colmax_j(|B|) * K)  <=  K-independent bound of the split,
and, for the benchmark's input class (U[0,1), no cancellation), the usual (|A||B|)_ij-scaled error <= 1e-10."""
import ctypes as C

import numpy as np
import pytest

from marlin_b200 import _native as nat
from tests.harness import gpu  # noqa: F401  (a fixture)

pytestmark = pytest.mark.gpu


def run(gpu, A, B, slices, C0=None, mode=1):
    import torch
    lib, ctx = gpu
    m, k = A.shape
    n = B.shape[1]
    dA = torch.from_numpy(np.ascontiguousarray(A.T)).cuda()      # column-major storage
    dB = torch.from_numpy(np.ascontiguousarray(B.T)).cuda()
    dC = torch.from_numpy(np.ascontiguousarray(C0.T)).cuda() if C0 is not None else torch.full((n, m), float("nan"), dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    nat.check(lib.mb_set_fp64_mode(ctx, mode if slices else 0, slices or 7))
    p = lambda t: C.c_void_p(t.data_ptr())
    nat.check(lib.mb_dgemm_device(ctx, b"N", b"N", m, n, k, 1.0, p(dA), m, p(dB), k, 1.0 if C0 is not None else 0.0, p(dC), m))
    nat.check(lib.mb_synchronize(ctx))
    nat.check(lib.mb_set_fp64_mode(ctx, 0, 7))
    return dC.cpu().numpy().T


@pytest.mark.parametrize("shape", [(256, 256, 256), (384, 512, 640), (300, 520, 700), (1024, 768, 2048), (257, 259, 261)])
@pytest.mark.parametrize("slices", [6, 7, 8])
def test_int8_split_gemm_uniform_inputs(gpu, shape, slices):
    m, n, k = shape
    rng = np.random.default_rng(m + n + k)
    A, B = rng.random((m, k)), rng.random((k, n))          # the benchmark's input class: U[0,1)
    ref = A @ B
    got = run(gpu, A, B, slices)
    err = (np.abs(got - ref) / (np.abs(A) @ np.abs(B))).max()
    assert err <= {6: 2e-11, 7: 2e-13, 8: 5e-15}[slices], err
    assert np.linalg.norm(got - ref) / np.linalg.norm(ref) <= 1e-10


@pytest.mark.parametrize("shape", [(256, 256, 256), (300, 520, 700), (1024, 768, 2048)])
@pytest.mark.parametrize("slices", [5, 6])
def test_int8_split_8bit_digits(gpu, shape, slices):
    """8-bit digit planes (MB_FP64_INT8_SPLIT8): 5 planes = 38 fractional bits in 15 int8 GEMMs."""
    m, n, k = shape
    rng = np.random.default_rng(m * 3 + n + k)
    A, B = rng.random((m, k)), rng.random((k, n))
    ref = A @ B
    got = run(gpu, A, B, slices, mode=2)
    err = (np.abs(got - ref) / (np.abs(A) @ np.abs(B))).max()
    assert err <= {5: 5e-11, 6: 5e-13}[slices], err
    As = (rng.random((m, k)) - 0.5)
    Bs = (rng.random((k, n)) - 0.5)
    got = run(gpu, As, Bs, slices, mode=2)
    scale = np.abs(As).max(axis=1)[:, None] * np.abs(Bs).max(axis=0)[None, :] * k
    assert (np.abs(got - As @ Bs) / scale).max() <= {5: 1e-11, 6: 1e-13}[slices]


def test_int8_split_signed_scaled_rows_and_accumulate(gpu):
    """Signed data, per-row / per-column magnitudes spread over 2^-40..2^40 (exact power-of-two scaling must absorb them),
    zero rows/columns, and C += A*B."""
    rng = np.random.default_rng(7)
    m, n, k = 512, 384, 1024
    A = (rng.random((m, k)) - 0.5) * np.exp2(rng.integers(-40, 40, size=(m, 1)))
    B = (rng.random((k, n)) - 0.5) * np.exp2(rng.integers(-40, 40, size=(1, n)))
    A[5, :] = 0.0
    B[:, 9] = 0.0
    C0 = rng.random((m, n))
    ref = A @ B
    got = run(gpu, A, B, 7)
    scale = np.abs(A).max(axis=1)[:, None] * np.abs(B).max(axis=0)[None, :] * k
    scale[scale == 0] = 1.0
    assert (np.abs(got - ref) / scale).max() <= 1e-13
    assert np.all(got[5, :] == 0.0) and np.all(got[:, 9] == 0.0)
    got2 = run(gpu, A, B, 7, C0=C0)
    assert (np.abs(got2 - (C0 + ref)) / (scale + np.abs(C0))).max() <= 1e-13


def test_native_mode_is_default_and_small_blocks_stay_native(gpu):
    rng = np.random.default_rng(3)
    A, B = rng.random((64, 64)), rng.random((64, 64))
    native = run(gpu, A, B, 0)
    split_requested = run(gpu, A, B, 7)          # below the 256 threshold -> DMMA kernel, bit-identical
    assert np.array_equal(native, split_requested)


@pytest.mark.parametrize("cfg", [(6, 1), (7, 1), (5, 2)])
def test_int8_split_equals_exact_integer_model_bit_for_bit(gpu, cfg):
    """Every step of the split is exact integer arithmetic (digit GEMMs accumulate in int32) and the groups are folded
    into C in a fixed order with one fp64 rounding each, so the kernel's result is fully determined:
    oracle/ozaki_model.py computes the same thing with numpy int64 and must agree to the last bit."""
    from oracle import ozaki_model as om
    slices, mode = cfg
    rng = np.random.default_rng(slices)
    A = (rng.random((300, 520)) - 0.3) * np.exp2(rng.integers(-6, 6, size=(300, 1)))
    B = (rng.random((520, 700)) - 0.3) * np.exp2(rng.integers(-6, 6, size=(1, 700)))
    want, _ = om.gemm(A, B, slices, 7 if mode == 1 else 8)
    got = run(gpu, A, B, slices, mode=mode)
    assert np.array_equal(got, want)
    C0 = rng.standard_normal((300, 700))
    want2, _ = om.gemm(A, B, slices, 7 if mode == 1 else 8, C0=C0)
    assert np.array_equal(run(gpu, A, B, slices, C0=C0, mode=mode), want2)

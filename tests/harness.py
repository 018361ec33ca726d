"""Plumbing shared by the test modules (not itself a test module): the SASS of the built library, the compiled C++ test
programs of the host mirror (tests/cpp), and a C ABI context for the modules that drive the library through ctypes."""
import collections
import ctypes as C
import functools
import re
import shutil
import subprocess
from pathlib import Path

import pytest

from marlin_b200 import _native as nat

ROOT = Path(__file__).resolve().parents[1]
BIN = ROOT / "scripts" / "bin"

# /*0a30*/  @!P0  DMMA.8x8x4 R24, R152, R160, R24 ;  ->  (0xa30, "DMMA.8x8x4", " R24, R152, R160, R24 ")
_INSTR = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Za-z0-9_.]*)([^;]*);")


@functools.cache
def sass() -> dict:
    """{mangled kernel name: [(address, opcode, operands), ...]} from one cuobjdump -sass of libmarlin_b200.so per
    process (no GPU needed); skips when cuobjdump cannot read the library.  Every kernel is sm_90a code."""
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    nat.load()
    out = subprocess.run([exe, "-sass", str(nat._LIB_PATH)], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=600)
    if out.returncode != 0:
        pytest.skip("cuobjdump unavailable: " + out.stderr[:200])
    assert set(re.findall(r"arch = (\w+)", out.stdout)) == {"sm_90a"}
    res = {}
    for chunk in re.split(r"\n\s*Function : ", out.stdout)[1:]:
        mangled = chunk.split("\n", 1)[0].strip()
        res[mangled] = [(int(a, 16), op, rest) for a, op, rest in _INSTR.findall(chunk)]
    return res


def family(needle: str) -> dict:
    """The kernels whose mangled name contains needle; there is at least one."""
    fam = {k: v for k, v in sass().items() if needle in k}
    assert fam, needle
    return fam


def ops(instrs) -> collections.Counter:
    """Full opcodes ("DMMA.8x8x4", "LDG.E.128", ...) and how often each occurs."""
    return collections.Counter(op for _, op, _ in instrs)


def count(ops: collections.Counter, prefix: str) -> int:
    """How many instructions have the base opcode prefix, whatever their modifiers."""
    return sum(v for k, v in ops.items() if k.split(".")[0] == prefix)


def body(instrs) -> list:
    """The kernel body: the instructions before the first CALL target, where the out-of-line subroutines begin."""
    targets = [int(m.group(1), 16) for _, op, rest in instrs if op.startswith("CALL") for m in [re.search(r"0x([0-9a-f]+)", rest)] if m]
    assert targets, "no CALL: nothing is out of line"
    return [i for i in instrs if i[0] < min(targets)]


def build_cpp(source: str, *, opt: str = "-O1", extra=()) -> Path:
    """Compile tests/cpp/<source>.cpp against the C ABI and the host mirror (include/) with plain g++ and -Werror into
    scripts/bin/<source>; the compiler's output is the assertion message when it fails."""
    nat.load()
    exe = BIN / source
    BIN.mkdir(parents=True, exist_ok=True)
    cmd = [shutil.which("g++") or "g++", "-std=c++17", opt, "-Wall", "-Werror", *extra, f"-I{ROOT / 'include'}",
           str(ROOT / "tests" / "cpp" / f"{source}.cpp"), f"-L{ROOT / 'marlin_b200' / 'lib'}", "-lmarlin_b200",
           "-Wl,-rpath,$ORIGIN/../../marlin_b200/lib", "-o", str(exe)]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert out.returncode == 0, out.stdout
    return exe


def run_cpp(exe: Path, *args, timeout: float = 300, status: int = 0) -> str:
    """Run a compiled test program, assert its exit status and return its output."""
    out = subprocess.run([str(exe), *map(str, args)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=timeout)
    assert out.returncode == status, out.stdout[-3000:]
    return out.stdout


def no_gpu_check(exe: Path, *args) -> None:
    """Without a GPU the program exits with status 3 and the library's "no CPU fallback" error."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the module's GPU test runs this program")
    assert "no CPU fallback" in run_cpp(exe, *args, timeout=120, status=3)


@pytest.fixture(scope="module")
def gpu():
    """(lib, ctx): a C ABI context on device 0 for the module, back in native fp64 mode before it shuts down."""
    lib = nat.load()
    ctx = nat.c_ctx()
    nat.check(lib.mb_init(0, C.byref(ctx)))
    yield lib, ctx
    lib.mb_set_fp64_mode(ctx, 0, 7)
    lib.mb_shutdown(ctx)

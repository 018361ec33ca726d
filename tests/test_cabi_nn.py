"""The NeuralNetwork entries of the C ABI: declared in include/marlin_b200.h, exported by the library, bound in _native."""
import re
from pathlib import Path

from marlin_b200 import _native as nat

ROOT = Path(__file__).resolve().parents[1]
ENTRIES = {"mb_nn_labels_upload", "mb_nn_labels_free", "mb_nn_gradient", "mb_nn_step"}


def test_nn_entries_are_declared_exported_and_bound():
    lib = nat.load()
    header = (ROOT / "include" / "marlin_b200.h").read_text()
    assert {n for n in re.findall(r"\b(mb_nn_[a-z0-9_]+)\s*\(", header)} == ENTRIES
    for name in ENTRIES:
        assert hasattr(lib, name) and name in nat.SIGNATURES

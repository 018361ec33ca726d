"""The JVM side of sparse blocks: every sparse native of Native.scala has its JNI twin (checked for all natives by
test_jni_veneer.py) and is called from the Scala host sources, and the Scala SubMatrix has the reference's sparse
surface (matrix/SubMatrix.scala:22-25, 39)."""
import re
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
SCALA = ROOT / "scala"
SPARSE_NATIVES = ("sparseUpload", "sparseDownload", "sparseNnz", "sparseAlloc", "sparseFree", "sparseValuesOp", "sparseToDense",
                  "spmmDenseSparse", "spmmSparseDense", "spgemm", "sparseColumnCount", "fillSparseUniform")


def test_every_sparse_native_is_declared_bound_and_called():
    native = (SCALA / "edu" / "nju" / "pasalab" / "marlin" / "matrix" / "Native.scala").read_text()
    jni = (ROOT / "jni" / "marlin_b200_jni.c").read_text()
    used = set()
    for f in SCALA.rglob("*.scala"):
        if f.name != "Native.scala":
            used |= set(re.findall(r"\bNative\.(\w+)", f.read_text()))
    for name in SPARSE_NATIVES:
        assert re.search(rf"@native\s+def\s+{name}\s*\(", native), name
        assert f"NATIVE(" in jni and re.search(rf"NATIVE\(\w+, {name}\)", jni), name
        assert name in used, f"{name} is never called from Scala"


def test_scala_submatrix_has_the_sparse_surface():
    text = (SCALA / "edu" / "nju" / "pasalab" / "marlin" / "matrix" / "SubMatrix.scala").read_text()
    assert "def this(spMatrix: SparseMatrix)" in text
    assert "def isSparse: Boolean = sparseHandle != 0L" in text
    assert "def isSparse: Boolean = false" not in text and "keep their JVM implementation" not in text

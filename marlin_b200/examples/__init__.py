"""Command-line drivers of the multiply path, taking the same positional arguments as the reference's example mains
(examples/MatrixMultiply.scala, BLAS3.scala, RMMcompare.scala): `python -m marlin_b200.examples.matrix_multiply 16384 16384
16384 8` on one GPU, or under `torchrun --nproc-per-node N` with one process per GPU.  PageRank's loader and loop are also
callable as functions (examples/PageRank.scala)."""
from .page_rank import loadLinksMatrix, pageRank  # noqa: F401

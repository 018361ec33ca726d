"""Command-line drivers of the multiply path, taking the same positional arguments as the reference's example mains
(examples/MatrixMultiply.scala, BLAS3.scala, RMMcompare.scala): `python -m marlin_b200.examples.matrix_multiply 16384 16384
16384 8` on one GPU, or under `torchrun --nproc-per-node N` with one process per GPU.  PageRank's loader and loop are also
callable as functions (examples/PageRank.scala), and so are NeuralNetwork's (examples/NeuralNetwork.scala,
`examples.neural_network`)."""
from . import neural_network  # noqa: F401
from .page_rank import loadLinksMatrix, pageRank  # noqa: F401

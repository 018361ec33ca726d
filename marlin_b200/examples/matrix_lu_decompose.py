"""examples/MatrixLUDecompose.scala — `matrix_lu_decompose <input path> <rows> <cols> <output path> <cores>`: the block LU
decomposition of a matrix read from `row:v,v,...` lines, saved as the packed L (unit lower) and U in DenseVecMatrix
format.  luDecompose() runs in "auto" mode: "dist" (sharded across the ranks) above 6000 rows, one device call below.
<rows>, <cols> and <cores> complete the reference's argument list; the matrix's dimensions come from the file."""
import sys

from ._common import start, stop


def main(args):
    if len(args) < 5:
        print("arguments wrong, the arguments should be <input path> <row number of the matrix> "
              "<column number of the matrix> <output path> <cores across the cluster>", file=sys.stderr)
        sys.exit(-1)
    mb, _ = start()
    mat = mb.MTUtils.loadMatrixFile(None, args[0])
    lu, _ = mat.luDecompose()
    lu.saveToFileSystem(args[3])
    stop()


if __name__ == "__main__":
    main(sys.argv[1:])

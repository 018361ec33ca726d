"""examples/SparseMultiply.scala:10-81 — `sparse_multiply <A rows> <A cols / B rows> <B cols> <density> <mode> [<seed>]`:
BlockMatrix multiplies on a 6 x 6 grid with sparse blocks (modes 3 to 6).  Modes 1 and 2 need SparseVecMatrix, which
this library does not have."""
import sys
import time

from ._common import start, stop

MODES = {
    1: "SparseVecMatrix multiply SparseVecMatrix with CRM algorithm",
    2: "SparseVecMatrix multiply SparseVecMatrix with sparse to dense vector",
    3: "BlockMatrix multiply BlockMatrix with sparse format",
    4: "BlockMatrix multiply BlockMatrix with dense format",
    5: "Dense BlockMatrix multiply Sparse BlockMatrix with dense-sparse format",
    6: "Dense BlockMatrix multiply Sparse BlockMatrix with dense-dense format",
}


def main(args):
    if len(args) < 5:
        sys.stderr.write("usage: sparse_multiply <matrixA row length> <matrixA column length> <matrixB column length> "
                         "<density> <mode> [<seed>]\n")
        for m, text in MODES.items():
            sys.stderr.write(f"mode {m}: {text}\n")
        sys.exit(1)
    rowA, colA, colB, density, mode = int(args[0]), int(args[1]), int(args[2]), float(args[3]), int(args[4])
    seed = int(args[5]) if len(args) > 5 else None
    if mode in (1, 2):
        print(f"mode {mode} ({MODES[mode]}) is not supported: SparseVecMatrix is not part of marlin_b200")
        return
    mb, rank = start()
    rnd = mb.MTUtils.randomBlockMatrix
    s2 = None if seed is None else seed + 1
    if mode == 3:
        A, B = rnd(None, rowA, colA, 6, 6, (True, density), seed=seed), rnd(None, colA, colB, 6, 6, (True, density), seed=s2)
    elif mode == 4:
        A = rnd(None, rowA, colA, 6, 6, (True, density), seed=seed).toDenseBlocks()
        B = rnd(None, colA, colB, 6, 6, (True, density), seed=s2).toDenseBlocks()
    elif mode == 5:
        A, B = rnd(None, rowA, colA, 6, 6, seed=seed), rnd(None, colA, colB, 6, 6, (True, density), seed=s2)
    elif mode == 6:
        A = rnd(None, rowA, colA, 6, 6, seed=seed)
        B = rnd(None, colA, colB, 6, 6, (True, density), seed=s2).toDenseBlocks()
    else:
        raise SystemExit(f"unknown mode {mode}")
    mb.MTUtils.evaluate(A)
    t0 = time.perf_counter()
    result = A.multiply(B)
    count = result.elementsCount()
    mb.MTUtils.evaluate(result)
    if rank == 0:
        print(f"result blocks count: {count}")
        print(f"{MODES[mode]} used time: {(time.perf_counter() - t0) * 1e3:.1f} ms")
    stop()


if __name__ == "__main__":
    main(sys.argv[1:])

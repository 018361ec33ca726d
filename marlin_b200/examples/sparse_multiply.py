"""examples/SparseMultiply.scala:10-81 — `sparse_multiply <A rows> <A cols / B rows> <B cols> <density> <mode> [<seed>]`:
mode 1 multiplies two random SparseVecMatrix row by row into a CoordinateMatrix (multiplySparse) and prints its entries
count; mode 2 densifies the same two matrices and multiplies them as DenseVecMatrix on a 6 x 6 x 6 split; modes 3 to 6
are BlockMatrix multiplies on a 6 x 6 grid with sparse blocks."""
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


def _entries_count(result) -> int:
    """entries.count(): every rank's entries (an object gather, which NCCL-only groups support)."""
    from ..runtime import world
    _, ws = world()
    if ws == 1:
        return len(result.rows)
    import torch.distributed as dist
    counts = [None] * ws
    dist.all_gather_object(counts, len(result.rows))
    return sum(counts)


def main(args):
    if len(args) < 5:
        sys.stderr.write("usage: sparse_multiply <matrixA row length> <matrixA column length> <matrixB column length> "
                         "<density> <mode> [<seed>]\n")
        for m, text in MODES.items():
            sys.stderr.write(f"mode {m}: {text}\n")
        sys.exit(1)
    rowA, colA, colB, density, mode = int(args[0]), int(args[1]), int(args[2]), float(args[3]), int(args[4])
    seed = int(args[5]) if len(args) > 5 else None
    mb, rank = start()
    if mode in (1, 2):
        s2 = None if seed is None else seed + 1
        A = mb.MTUtils.randomSpaVecMatrix(None, rowA, colA, density, seed=seed)
        B = mb.MTUtils.randomSpaVecMatrix(None, colA, colB, density, seed=s2)
        if mode == 1:
            t0 = time.perf_counter()
            result = A.multiplySparse(B)
            count = _entries_count(result)
            if rank == 0:
                print(f"result entries count: {count}")
                print(f"sparse-multiply used time: {(time.perf_counter() - t0) * 1e3:.1f} ms")
        else:
            denA, denB = A.toDenseVecMatrix(), B.toDenseVecMatrix()
            mb.MTUtils.evaluate(denB)
            t0 = time.perf_counter()
            result = denA.multiply(denB, (6, 6, 6))
            count = result.elementsCount()
            mb.MTUtils.evaluate(result)
            if rank == 0:
                print(f"result blocks count: {count}")
                print(f"dense-multiply used time: {(time.perf_counter() - t0) * 1e3:.1f} ms")
        stop()
        return
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

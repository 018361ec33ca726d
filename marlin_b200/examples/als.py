"""examples/ALS.scala:9-28 — `als <input> <rank> <iteration> <lambda> {<numUserBlock> <numProductBlock>}`: load a
coordinate file (`row col value [timestamp]`, e.g. MovieLens ratings) and factorise it with CoordinateMatrix.ALS."""
import sys

from ._common import millis, start, stop


def main(args):
    if len(args) < 3:
        print("Usage: ALS <input> <rank> <iteration> <lambda> {<numUserBlock> <numProductBlock>}", file=sys.stderr)
        sys.exit(1)
    mb, rank = start()
    path, rnk, iterations, lam = args[0], int(args[1]), int(args[2]), float(args[3])
    num_user_block = int(args[4]) if len(args) > 4 else 10
    num_product_block = int(args[5]) if len(args) > 5 else 10
    rating_matrix = mb.MTUtils.loadCoordinateMatrix(None, path)
    t0 = millis()
    user_factor, product_factor = rating_matrix.ALS(rnk, iterations, lam, num_user_block, num_product_block)
    used = millis() - t0
    users = sum(user_factor._gather([len(user_factor.ids)]))            # userFactor.getRows.count()
    products = sum(product_factor._gather([len(product_factor.ids)]))   # productFactor.getRows.count()
    if rank == 0:
        print(f"{users} user factors, {products} product factors of rank {rnk}; {iterations} iterations used time {used:.0f} millis")
    stop()


if __name__ == "__main__":
    main(sys.argv[1:])

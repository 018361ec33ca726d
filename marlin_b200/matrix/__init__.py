from .block import BlockID
from .block_matrix import BlockMatrix
from .coordinate_matrix import CoordinateMatrix
from .dense_vec_matrix import DenseVecMatrix
from .distributed_matrix import DistributedMatrix
from .distributed_vector import DistributedVector
from .sparse_matrix import SparseMatrix, SparseVector
from .sparse_vec_matrix import SparseVecMatrix
from .sub_matrix import SubMatrix

__all__ = ["BlockID", "BlockMatrix", "CoordinateMatrix", "DenseVecMatrix", "DistributedMatrix", "DistributedVector", "SparseMatrix", "SparseVector",
           "SparseVecMatrix", "SubMatrix"]

"""DistributedMatrix — the trait that is the drop-in API contract (matrix/DistributedMatrix.scala:9-76)."""
from __future__ import annotations


class DistributedMatrix:
    def numRows(self) -> int:
        raise NotImplementedError

    def numCols(self) -> int:
        raise NotImplementedError

    def add(self, other):
        raise NotImplementedError

    def subtract(self, other):
        raise NotImplementedError

    def multiply(self, other, *args, **kwargs):
        raise NotImplementedError

    def divide(self, b):
        raise NotImplementedError

    def sum(self) -> float:
        raise NotImplementedError

    def dotProduct(self, other):
        raise NotImplementedError

    def transpose(self):
        raise NotImplementedError

    def cBind(self, other):
        """:63 — this matrix with the columns of `other` appended."""
        raise NotImplementedError

    def toBreeze(self):
        raise NotImplementedError

    def saveToFileSystem(self, path: str):
        raise NotImplementedError

    def print(self) -> None:
        raise NotImplementedError

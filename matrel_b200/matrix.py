"""Host-side block types mirroring the reference data model
(<reference>/src/main/scala/org/apache/spark/sql/matfast/matrix/MLMatrix.scala):
``DenseMatrix`` (:234-241), ``SparseMatrix`` (:525-543), ``MatrixBlock`` (:1205).

These are plain containers for moving blocks across the C ABI (the 7-field struct of
MLMatrixSerializer.scala:26-48).  They carry no arithmetic: every operator runs on the GPU.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Union

import numpy as np


class DenseMatrix:
    """numRows x numCols doubles, column-major; row-major when ``isTransposed`` (MLMatrix.scala:216-231)."""

    def __init__(self, numRows: int, numCols: int, values, isTransposed: bool = False):
        self.numRows = int(numRows)
        self.numCols = int(numCols)
        self.values = np.ascontiguousarray(values, dtype=np.float64).reshape(-1)
        self.isTransposed = bool(isTransposed)

    def transpose(self) -> "DenseMatrix":
        """Metadata only, shares ``values`` (MLMatrix.scala:312)."""
        return DenseMatrix(self.numCols, self.numRows, self.values, not self.isTransposed)

    def to_numpy(self) -> np.ndarray:
        """Logical numRows x numCols view of the stored values."""
        if not self.isTransposed:
            return self.values.reshape(self.numCols, self.numRows).T
        return self.values.reshape(self.numRows, self.numCols)

    @staticmethod
    def from_numpy(a: np.ndarray, transposed_storage: bool = False) -> "DenseMatrix":
        a = np.asarray(a, dtype=np.float64)
        if transposed_storage:
            return DenseMatrix(a.shape[0], a.shape[1], np.ascontiguousarray(a).reshape(-1), True)
        return DenseMatrix(a.shape[0], a.shape[1], np.ascontiguousarray(a.T).reshape(-1), False)

    def __repr__(self) -> str:
        return f"DenseMatrix({self.numRows}x{self.numCols}, isTransposed={self.isTransposed})"


class SparseMatrix:
    """CSC (CSR when ``isTransposed``) block (MLMatrix.scala:501-543)."""

    def __init__(self, numRows: int, numCols: int, colPtrs, rowIndices, values, isTransposed: bool = False):
        self.numRows = int(numRows)
        self.numCols = int(numCols)
        self.colPtrs = np.ascontiguousarray(colPtrs, dtype=np.int32).reshape(-1)
        self.rowIndices = np.ascontiguousarray(rowIndices, dtype=np.int32).reshape(-1)
        self.values = np.ascontiguousarray(values, dtype=np.float64).reshape(-1)
        self.isTransposed = bool(isTransposed)

    def transpose(self) -> "SparseMatrix":
        """Metadata only (MLMatrix.scala:634-635)."""
        return SparseMatrix(self.numCols, self.numRows, self.colPtrs, self.rowIndices, self.values,
                            not self.isTransposed)

    def to_numpy(self) -> np.ndarray:
        out = np.zeros((self.numRows, self.numCols))
        major = np.repeat(np.arange(self.colPtrs.size - 1), np.diff(self.colPtrs))
        if not self.isTransposed:
            out[self.rowIndices, major] = self.values
        else:
            out[major, self.rowIndices] = self.values
        return out

    def __repr__(self) -> str:
        return (f"SparseMatrix({self.numRows}x{self.numCols}, nnz={self.values.size}, "
                f"isTransposed={self.isTransposed})")


MLMatrix = Union[DenseMatrix, SparseMatrix]


@dataclass
class MatrixBlock:
    """One Dataset row ``(rid, cid, matrix)`` (MLMatrix.scala:1205)."""
    rid: int
    cid: int
    matrix: MLMatrix

"""Lazy logical plans + the algebraic rewrites of the reference's planner, above the C ABI.

The reference builds one logical node per ``Dataset`` call (M/plans/MatrixOperator.scala:25-166) and
``MatrixOperators.apply`` (M/execution/MatfastPlanner.scala:42-279) maps them to physical operators,
pushing aggregates through their children on the way -- e.g. ``trace(A B) -> sum(A^T o B)`` (:238-241),
``sum(A B) -> colSum(A) . rowSum(B)`` (:220-225), ``rowSum(A B) -> A . rowSum(B)`` (:181-185) -- which
turns O(N^3) queries into O(N^2) ones.  This module restates that strategy: ``LazyDataset`` records
nodes, ``execute()`` walks them with the same case analysis and runs the chosen physical operators
eagerly through ``matrel_b200.dataset.Dataset`` (i.e. the sm_90a kernels).

M/ = <reference>/src/main/scala/org/apache/spark/sql/matfast/
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional

from .dataset import Dataset


# ---- logical nodes (M/plans/MatrixOperator.scala) -------------------------------------------------------
@dataclass
class Leaf:
    ds: Dataset


@dataclass
class ProjectOperator:              # :25-33
    child: object
    nrows: int
    ncols: int
    blkSize: int
    rowOrCol: bool
    index: int


@dataclass
class SelectOperator:               # :35-41
    child: object
    nrows: int
    ncols: int
    blkSize: int
    rowIdx: int
    colIdx: int


@dataclass
class TransposeOperator:            # :43-45
    child: object


@dataclass
class RowSumOperator:               # :47-51
    child: object
    nrows: int
    ncols: int


@dataclass
class ColumnSumOperator:            # :53-57
    child: object
    nrows: int
    ncols: int


@dataclass
class SumOperator:                  # :59-63
    child: object
    nrows: int
    ncols: int


@dataclass
class TraceOperator:                # :65-69
    child: object
    nrows: int
    ncols: int


@dataclass
class MatrixScalarAddOperator:      # :77-79
    child: object
    alpha: float


@dataclass
class MatrixScalarMultiplyOperator:  # :81-83
    child: object
    alpha: float


@dataclass
class MatrixPowerOperator:          # :85-87
    child: object
    alpha: float


@dataclass
class _Binary:
    left: object
    leftRowNum: int
    leftColNum: int
    right: object
    rightRowNum: int
    rightColNum: int
    blkSize: int


class MatrixElementAddOperator(_Binary):            # :95-107
    pass


class MatrixElementMultiplyOperator(_Binary):       # :109-121
    pass


class MatrixElementDivideOperator(_Binary):         # :123-135
    pass


class MatrixMatrixMultiplicationOperator(_Binary):  # :137-149
    pass


class RankOneUpdateOperator(_Binary):               # :153-166
    pass


# ---- planner + executor (M/execution/MatfastPlanner.scala:42-279) ------------------------------------------
class Planner:
    """``run(node)`` = ``planLater(node).execute()``; ``trace`` lists the physical operators it chose."""

    def __init__(self, rewrite: bool = True):
        self.rewrite = rewrite
        self.trace: List[str] = []

    def _phys(self, name: str):
        self.trace.append(name)

    def run(self, n) -> Dataset:
        R = self.run
        if isinstance(n, Leaf):
            return n.ds
        if isinstance(n, ProjectOperator):                                     # :44-124
            c = n.child
            P = lambda ch, nr, nc: ProjectOperator(ch, nr, nc, n.blkSize, n.rowOrCol, n.index)  # noqa: E731
            if self.rewrite:
                if isinstance(c, TransposeOperator):      # a row of A^T is a column of A (the reference emits it un-transposed)
                    self._phys("ProjectColumnDirectExecution" if n.rowOrCol else "ProjectRowDirectExecution")
                    return R(c.child).project(n.ncols, n.nrows, n.blkSize, not n.rowOrCol, n.index).transpose()
                if isinstance(c, MatrixScalarAddOperator):
                    self._phys("MatrixScalarAddExecution")
                    return R(P(c.child, n.nrows, n.ncols)).addScalar(c.alpha)
                if isinstance(c, MatrixScalarMultiplyOperator):
                    self._phys("MatrixScalarMultiplyExecution")
                    return R(P(c.child, n.nrows, n.ncols)).multiplyScalar(c.alpha)
                if isinstance(c, (MatrixElementAddOperator, MatrixElementMultiplyOperator, MatrixElementDivideOperator)):
                    fn = {MatrixElementAddOperator: "addElement", MatrixElementMultiplyOperator: "multiplyElement",
                          MatrixElementDivideOperator: "divideElement"}[type(c)]
                    self._phys(type(c).__name__.replace("Operator", "Execution"))
                    lr, lc = (1, c.leftColNum) if n.rowOrCol else (c.leftRowNum, 1)
                    rr, rc = (1, c.rightColNum) if n.rowOrCol else (c.rightRowNum, 1)
                    return getattr(R(P(c.left, c.leftRowNum, c.leftColNum)), fn)(
                        lr, lc, R(P(c.right, c.rightRowNum, c.rightColNum)), rr, rc, c.blkSize)
                if isinstance(c, MatrixMatrixMultiplicationOperator):          # row_i(A B) = row_i(A) B ; col_j(A B) = A col_j(B)
                    self._phys("MatrixMatrixMultiplicationExecution")
                    if n.rowOrCol:
                        return R(P(c.left, c.leftRowNum, c.leftColNum)).matrixMultiply(
                            1, c.leftColNum, R(c.right), c.rightRowNum, c.rightColNum, c.blkSize)
                    return R(c.left).matrixMultiply(c.leftRowNum, c.leftColNum, R(P(c.right, c.rightRowNum, c.rightColNum)),
                                                    c.rightRowNum, 1, c.blkSize)
            self._phys("ProjectRowDirectExecution" if n.rowOrCol else "ProjectColumnDirectExecution")
            return R(c).project(n.nrows, n.ncols, n.blkSize, n.rowOrCol, n.index)
        if isinstance(n, SelectOperator):                                      # :125-166
            c = n.child
            S = lambda ch, nr, nc: SelectOperator(ch, nr, nc, n.blkSize, n.rowIdx, n.colIdx)  # noqa: E731
            if self.rewrite:
                if isinstance(c, TransposeOperator):
                    self._phys("SelectDirectExecution")
                    return R(c.child).selection(n.ncols, n.nrows, n.blkSize, n.colIdx, n.rowIdx)
                if isinstance(c, MatrixScalarAddOperator):
                    self._phys("MatrixScalarAddExecution")
                    return R(S(c.child, n.nrows, n.ncols)).addScalar(c.alpha)
                if isinstance(c, MatrixScalarMultiplyOperator):
                    self._phys("MatrixScalarMultiplyExecution")
                    return R(S(c.child, n.nrows, n.ncols)).multiplyScalar(c.alpha)
                if isinstance(c, (MatrixElementAddOperator, MatrixElementMultiplyOperator, MatrixElementDivideOperator)):
                    fn = {MatrixElementAddOperator: "addElement", MatrixElementMultiplyOperator: "multiplyElement",
                          MatrixElementDivideOperator: "divideElement"}[type(c)]
                    self._phys(type(c).__name__.replace("Operator", "Execution"))
                    return getattr(R(S(c.left, c.leftRowNum, c.leftColNum)), fn)(
                        1, 1, R(S(c.right, c.rightRowNum, c.rightColNum)), 1, 1, c.blkSize)
                if isinstance(c, MatrixMatrixMultiplicationOperator):          # (A B)_ij = row_i(A) . col_j(B)
                    self._phys("MatrixMatrixMultiplicationExecution")
                    row = ProjectOperator(c.left, c.leftRowNum, c.leftColNum, n.blkSize, True, n.rowIdx)
                    col = ProjectOperator(c.right, c.rightRowNum, c.rightColNum, n.blkSize, False, n.colIdx)
                    return R(row).matrixMultiply(1, c.leftColNum, R(col), c.rightRowNum, 1, c.blkSize)
            self._phys("SelectDirectExecution")
            return R(c).selection(n.nrows, n.ncols, n.blkSize, n.rowIdx, n.colIdx)
        if isinstance(n, TransposeOperator):                                   # :167
            self._phys("MatrixTransposeExecution")
            return R(n.child).transpose()
        if isinstance(n, RowSumOperator):                                      # :168-187
            c = n.child
            if self.rewrite:
                if isinstance(c, TransposeOperator):
                    self._phys("MatrixTransposeExecution")
                    return R(ColumnSumOperator(c.child, n.ncols, n.nrows)).transpose()
                if isinstance(c, MatrixScalarAddOperator):
                    self._phys("MatrixScalarAddExecution")
                    return R(RowSumOperator(c.child, n.nrows, n.ncols)).addScalar(c.alpha * n.ncols)
                if isinstance(c, MatrixScalarMultiplyOperator):
                    self._phys("MatrixScalarMultiplyExecution")
                    return R(RowSumOperator(c.child, n.nrows, n.ncols)).multiplyScalar(c.alpha)
                if isinstance(c, MatrixElementAddOperator):
                    self._phys("MatrixElementAddExecution")
                    return R(RowSumOperator(c.left, c.leftRowNum, c.leftColNum)).addElement(
                        c.leftRowNum, 1, R(RowSumOperator(c.right, c.rightRowNum, c.rightColNum)), c.rightRowNum, 1, c.blkSize)
                if isinstance(c, MatrixMatrixMultiplicationOperator):
                    self._phys("MatrixMatrixMultiplicationExecution")
                    return R(c.left).matrixMultiply(c.leftRowNum, c.leftColNum,
                                                    R(RowSumOperator(c.right, c.rightRowNum, c.rightColNum)),
                                                    c.rightRowNum, 1, c.blkSize)
            self._phys("RowSumDirectExecution")
            return R(c).rowSum(n.nrows, n.ncols)
        if isinstance(n, ColumnSumOperator):                                   # :188-208
            c = n.child
            if self.rewrite:
                if isinstance(c, TransposeOperator):
                    self._phys("MatrixTransposeExecution")
                    return R(RowSumOperator(c.child, n.ncols, n.nrows)).transpose()
                if isinstance(c, MatrixScalarAddOperator):
                    self._phys("MatrixScalarAddExecution")
                    return R(ColumnSumOperator(c.child, n.nrows, n.ncols)).addScalar(c.alpha * n.nrows)
                if isinstance(c, MatrixScalarMultiplyOperator):
                    self._phys("MatrixScalarMultiplyExecution")
                    return R(ColumnSumOperator(c.child, n.nrows, n.ncols)).multiplyScalar(c.alpha)
                if isinstance(c, MatrixElementAddOperator):
                    self._phys("MatrixElementAddExecution")
                    return R(ColumnSumOperator(c.left, c.leftRowNum, c.leftColNum)).addElement(
                        1, c.leftColNum, R(ColumnSumOperator(c.right, c.rightRowNum, c.rightColNum)), 1, c.rightColNum, c.blkSize)
                if isinstance(c, MatrixMatrixMultiplicationOperator):
                    self._phys("MatrixMatrixMultiplicationExecution")
                    return R(ColumnSumOperator(c.left, c.leftRowNum, c.leftColNum)).matrixMultiply(
                        1, c.leftColNum, R(c.right), c.rightRowNum, c.rightColNum, c.blkSize)
            self._phys("ColumnSumDirectExecution")
            return R(c).colSum(n.nrows, n.ncols)
        if isinstance(n, SumOperator):                                         # :209-227
            c = n.child
            if self.rewrite:
                if isinstance(c, TransposeOperator):
                    self._phys("SumDirectExecution")
                    return R(c.child).sum(n.ncols, n.nrows)
                if isinstance(c, MatrixScalarAddOperator):
                    self._phys("MatrixScalarAddExecution")
                    return R(SumOperator(c.child, n.nrows, n.ncols)).addScalar(c.alpha * n.nrows * n.ncols)
                if isinstance(c, MatrixScalarMultiplyOperator):
                    self._phys("MatrixScalarMultiplyExecution")
                    return R(SumOperator(c.child, n.nrows, n.ncols)).multiplyScalar(c.alpha)
                if isinstance(c, MatrixElementAddOperator):
                    self._phys("MatrixElementAddExecution")
                    return R(SumOperator(c.left, c.leftRowNum, c.leftColNum)).addElement(
                        1, 1, R(SumOperator(c.right, c.rightRowNum, c.rightColNum)), 1, 1, c.blkSize)
                if isinstance(c, MatrixMatrixMultiplicationOperator):          # sum(A B) = colSum(A) . rowSum(B)
                    self._phys("MatrixMatrixMultiplicationExecution")
                    return R(ColumnSumOperator(c.left, c.leftRowNum, c.leftColNum)).matrixMultiply(
                        1, c.leftColNum, R(RowSumOperator(c.right, c.rightRowNum, c.rightColNum)), c.rightRowNum, 1, c.blkSize)
            self._phys("SumDirectExecution")
            return R(c).sum(n.nrows, n.ncols)
        if isinstance(n, TraceOperator):                                       # :228-244
            c = n.child
            if self.rewrite:
                if isinstance(c, TransposeOperator):
                    self._phys("TraceDirectExecution")
                    return R(c.child).trace(n.ncols, n.nrows)
                if isinstance(c, MatrixScalarAddOperator):
                    self._phys("MatrixScalarAddExecution")
                    return R(TraceOperator(c.child, n.nrows, n.ncols)).addScalar(c.alpha * n.nrows)
                if isinstance(c, MatrixScalarMultiplyOperator):
                    self._phys("MatrixScalarMultiplyExecution")
                    return R(TraceOperator(c.child, n.nrows, n.ncols)).multiplyScalar(c.alpha)
                if isinstance(c, MatrixElementAddOperator):
                    self._phys("MatrixElementAddExecution")
                    return R(TraceOperator(c.left, c.leftRowNum, c.leftColNum)).addElement(
                        1, 1, R(TraceOperator(c.right, c.rightRowNum, c.rightColNum)), 1, 1, c.blkSize)
                if isinstance(c, MatrixMatrixMultiplicationOperator):          # trace(A B) = sum(A^T o B)
                    self._phys("SumDirectExecution")
                    prod = MatrixElementMultiplyOperator(TransposeOperator(c.left), c.leftColNum, c.leftRowNum,
                                                         c.right, c.rightRowNum, c.rightColNum, c.blkSize)
                    return R(prod).sum(c.rightRowNum, c.rightColNum)
            self._phys("TraceDirectExecution")
            return R(c).trace(n.nrows, n.ncols)
        if isinstance(n, MatrixScalarAddOperator):                             # :245-246
            self._phys("MatrixScalarAddExecution")
            return R(n.child).addScalar(n.alpha)
        if isinstance(n, MatrixScalarMultiplyOperator):                        # :247-248
            self._phys("MatrixScalarMultiplyExecution")
            return R(n.child).multiplyScalar(n.alpha)
        if isinstance(n, MatrixPowerOperator):                                 # :249-250
            self._phys("MatrixPowerExecution")
            return R(n.child).power(n.alpha)
        if isinstance(n, _Binary):                                             # :253-276
            name, fn = {
                MatrixElementAddOperator: ("MatrixElementAddExecution", "addElement"),
                MatrixElementMultiplyOperator: ("MatrixElementMultiplyExecution", "multiplyElement"),
                MatrixElementDivideOperator: ("MatrixElementDivideExecution", "divideElement"),
                MatrixMatrixMultiplicationOperator: ("MatrixMatrixMultiplicationExecution", "matrixMultiply"),
                RankOneUpdateOperator: ("RankOneUpdateExecution", "matrixRankOneUpdate"),
            }[type(n)]
            self._phys(name)
            return getattr(R(n.left), fn)(n.leftRowNum, n.leftColNum, R(n.right), n.rightRowNum, n.rightColNum, n.blkSize)
        raise TypeError(f"no strategy for {n!r}")                              # `case _ => Nil`


class LazyDataset:
    """Lazy counterpart of ``Dataset``: the same method names (M/Dataset.scala:57-152) build nodes; nothing runs
    until an action (``execute`` / ``collect``), like the reference's ``QueryExecution`` (M/execution/QueryExecution.scala:32-40)."""

    def __init__(self, node):
        self.node = node

    @staticmethod
    def of(ds: Dataset) -> "LazyDataset":
        return LazyDataset(Leaf(ds))

    def _bin(self, cls, lr, lc, right, rr, rc, blk):
        return LazyDataset(cls(self.node, int(lr), int(lc), right.node, int(rr), int(rc), int(blk)))

    def matrixMultiply(self, lr, lc, right, rr, rc, blk):
        return self._bin(MatrixMatrixMultiplicationOperator, lr, lc, right, rr, rc, blk)

    def addElement(self, lr, lc, right, rr, rc, blk):
        return self._bin(MatrixElementAddOperator, lr, lc, right, rr, rc, blk)

    def multiplyElement(self, lr, lc, right, rr, rc, blk):
        return self._bin(MatrixElementMultiplyOperator, lr, lc, right, rr, rc, blk)

    def divideElement(self, lr, lc, right, rr, rc, blk):
        return self._bin(MatrixElementDivideOperator, lr, lc, right, rr, rc, blk)

    def matrixRankOneUpdate(self, lr, lc, right, rr, rc, blk):
        return self._bin(RankOneUpdateOperator, lr, lc, right, rr, rc, blk)

    def transpose(self):
        return LazyDataset(TransposeOperator(self.node))

    t = transpose

    def addScalar(self, alpha):
        return LazyDataset(MatrixScalarAddOperator(self.node, float(alpha)))

    def multiplyScalar(self, alpha):
        return LazyDataset(MatrixScalarMultiplyOperator(self.node, float(alpha)))

    def power(self, alpha):
        return LazyDataset(MatrixPowerOperator(self.node, float(alpha)))

    def project(self, nrows, ncols, blkSize, rowOrCol, index):
        return LazyDataset(ProjectOperator(self.node, int(nrows), int(ncols), int(blkSize), bool(rowOrCol), int(index)))

    def selection(self, nrows, ncols, blkSize, rowIdx, colIdx):
        return LazyDataset(SelectOperator(self.node, int(nrows), int(ncols), int(blkSize), int(rowIdx), int(colIdx)))

    def rowSum(self, nrows, ncols):
        return LazyDataset(RowSumOperator(self.node, int(nrows), int(ncols)))

    def colSum(self, nrows, ncols):
        return LazyDataset(ColumnSumOperator(self.node, int(nrows), int(ncols)))

    def sum(self, nrows, ncols):
        return LazyDataset(SumOperator(self.node, int(nrows), int(ncols)))

    def trace(self, nrows, ncols):
        if int(nrows) != int(ncols):                                           # Dataset.scala:80
            from ._native import IllegalArgumentException, MR_EDIM
            raise IllegalArgumentException(MR_EDIM, "requirement failed: Cannot perform trace() on a rectangle matrix")
        return LazyDataset(TraceOperator(self.node, int(nrows), int(ncols)))

    def execute(self, rewrite: bool = True, planner: Optional[Planner] = None) -> Dataset:
        return (planner or Planner(rewrite)).run(self.node)

    def collect(self):
        return self.execute().collect()

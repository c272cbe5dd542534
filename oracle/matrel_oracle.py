"""CPU oracle: a numpy restatement of the MatRel/MatFast block-matrix hot path.

TEST INFRASTRUCTURE ONLY.  Nothing in ``matrel_b200/`` may import this module; only
``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl reference``
legs use it, and only as the checker / reported CPU baseline (never as the product path).

PARITY UNPINNED: the reference ships no tests, golden vectors or published outputs for this
path (src/test/scala/.../basicOptSuites.scala:21-23 is an empty class) and it cannot be run
here (no JVM, no Spark jars).  The oracle is therefore pinned only against (i) the hand-derived
answers of the reference's println fixtures (example/BasicMatrixOps.scala:107-144,
matrix/LocalMatrix.scala:1096-1135; see tests/golden/) and (ii) an independent dense
``A_full @ B_full`` check.  The dense block product itself is netlib-java ``dgemm``
(com.github.fommil.netlib, resolved through spark-mllib 2.1.0, build.sbt:13; Spark 2.1.0 pins
netlib-java 1.1.2) -- standard BLAS semantics, restated here with ``numpy.matmul``.

All ``M/...`` citations are into
<reference>/src/main/scala/org/apache/spark/sql/matfast/.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Iterable, List, Optional, Tuple, Union

import numpy as np

# ----------------------------------------------------------------------------------------------
# Data model  (M/matrix/MLMatrix.scala)
# ----------------------------------------------------------------------------------------------


class IllegalArgumentException(ValueError):
    """Scala ``require`` failure: message is 'requirement failed: <msg>'."""


def require(cond: bool, msg: str) -> None:
    if not cond:
        raise IllegalArgumentException("requirement failed: " + msg)


class DenseMatrix:
    """M/matrix/MLMatrix.scala:234-241.  ``values`` column-major, or row-major when isTransposed."""

    def __init__(self, numRows: int, numCols: int, values, isTransposed: bool = False):
        values = np.ascontiguousarray(values, dtype=np.float64).reshape(-1)
        require(values.size == numRows * numCols,
                "The number of values supplied doesn't match the size of the matrix! "
                f"values.length: {values.size}, numRows * numCols: {numRows * numCols}")  # :240
        self.numRows, self.numCols = int(numRows), int(numCols)
        self.values = values
        self.isTransposed = bool(isTransposed)

    # M/matrix/MLMatrix.scala:285-289
    def index(self, i: int, j: int) -> int:
        require(0 <= i < self.numRows, f"Expected 0 <= i < {self.numRows}, got i = {i}.")
        require(0 <= j < self.numCols, f"Expected 0 <= j < {self.numCols}, got j = {j}.")
        return i + self.numRows * j if not self.isTransposed else j + self.numCols * i

    def apply(self, i: int, j: int) -> float:
        return float(self.values[self.index(i, j)])

    # M/matrix/MLMatrix.scala:312 -- metadata only, shares the backing array
    def transpose(self) -> "DenseMatrix":
        return DenseMatrix(self.numCols, self.numRows, self.values, not self.isTransposed)

    def to_numpy(self) -> np.ndarray:
        """Logical numRows x numCols array (a view when possible)."""
        if not self.isTransposed:
            return self.values.reshape(self.numCols, self.numRows).T
        return self.values.reshape(self.numRows, self.numCols)

    # M/matrix/MLMatrix.scala:55-61 -- always a fresh column-major array
    def toArray(self) -> np.ndarray:
        return np.ascontiguousarray(self.to_numpy().T).reshape(-1).copy()

    # M/matrix/MLMatrix.scala:353-374 -- CSC, isTransposed = false, drops exact zeros
    def toSparse(self) -> "SparseMatrix":
        a = self.to_numpy()
        colPtrs = [0]
        rowIndices: List[int] = []
        vals: List[float] = []
        for j in range(self.numCols):
            nz = np.nonzero(a[:, j] != 0.0)[0]
            rowIndices.extend(int(x) for x in nz)
            vals.extend(float(x) for x in a[nz, j])
            colPtrs.append(len(rowIndices))
        return SparseMatrix(self.numRows, self.numCols, colPtrs, rowIndices, vals)

    @staticmethod
    def zeros(numRows: int, numCols: int) -> "DenseMatrix":
        return DenseMatrix(numRows, numCols, np.zeros(numRows * numCols))

    @staticmethod
    def rand(numRows: int, numCols: int, rng: "JavaRandom") -> "DenseMatrix":
        """M/matrix/MLMatrix.scala:453-457: Array.fill(numRows*numCols)(rng.nextDouble())."""
        require(numRows * numCols <= 2**31 - 1,
                f"{numRows} x {numCols} dense matrix is too large to allocate")
        return DenseMatrix(numRows, numCols, rng.next_doubles(numRows * numCols))

    def __repr__(self) -> str:
        return f"DenseMatrix({self.numRows}x{self.numCols}, T={self.isTransposed})"


class SparseMatrix:
    """M/matrix/MLMatrix.scala:525-543.  CSC, or CSR when isTransposed."""

    def __init__(self, numRows, numCols, colPtrs, rowIndices, values, isTransposed: bool = False):
        colPtrs = np.ascontiguousarray(colPtrs, dtype=np.int32).reshape(-1)
        rowIndices = np.ascontiguousarray(rowIndices, dtype=np.int32).reshape(-1)
        values = np.ascontiguousarray(values, dtype=np.float64).reshape(-1)
        require(values.size == rowIndices.size,
                "The number of row indices and values don't match! "
                f"values.length: {values.size}, rowIndices.length: {rowIndices.size}")  # :533
        if isTransposed:
            require(colPtrs.size == numRows + 1,
                    f"Expecting {numRows + 1} colPtrs when numRows = {numRows} but got {colPtrs.size}")
        else:
            require(colPtrs.size == numCols + 1,
                    f"Expecting {numCols + 1} colPtrs when numCols = {numCols} but got {colPtrs.size}")
        require(values.size == int(colPtrs[-1]),
                "The last value of colPtrs must equal the number of elements. "
                f"values.length: {values.size}, colPtrs.last: {int(colPtrs[-1])}")  # :542
        self.numRows, self.numCols = int(numRows), int(numCols)
        self.colPtrs, self.rowIndices, self.values = colPtrs, rowIndices, values
        self.isTransposed = bool(isTransposed)

    # M/matrix/MLMatrix.scala:595-603 (binary search; negative when absent)
    def index(self, i: int, j: int) -> int:
        require(0 <= i < self.numRows, f"Expected 0 <= i < {self.numRows}, got i = {i}.")
        require(0 <= j < self.numCols, f"Expected 0 <= j < {self.numCols}, got j = {j}.")
        major, minor = (j, i) if not self.isTransposed else (i, j)
        lo, hi = int(self.colPtrs[major]), int(self.colPtrs[major + 1])
        seg = self.rowIndices[lo:hi]
        p = int(np.searchsorted(seg, minor))
        if p < seg.size and int(seg[p]) == minor:
            return lo + p
        return -(lo + p) - 1

    def apply(self, i: int, j: int) -> float:
        k = self.index(i, j)
        return 0.0 if k < 0 else float(self.values[k])

    # M/matrix/MLMatrix.scala:634-635
    def transpose(self) -> "SparseMatrix":
        return SparseMatrix(self.numCols, self.numRows, self.colPtrs, self.rowIndices,
                            self.values, not self.isTransposed)

    def to_numpy(self) -> np.ndarray:
        """foreachActive scatter (M/matrix/MLMatrix.scala:637-663); later duplicates overwrite."""
        out = np.zeros((self.numRows, self.numCols))
        nmajor = self.colPtrs.size - 1
        major = np.repeat(np.arange(nmajor), np.diff(self.colPtrs))
        if not self.isTransposed:
            out[self.rowIndices, major] = self.values
        else:
            out[major, self.rowIndices] = self.values
        return out

    def toArray(self) -> np.ndarray:
        return np.ascontiguousarray(self.to_numpy().T).reshape(-1).copy()

    # M/matrix/MLMatrix.scala:669-671
    def toDense(self) -> DenseMatrix:
        return DenseMatrix(self.numRows, self.numCols, self.toArray())

    def __repr__(self) -> str:
        return f"SparseMatrix({self.numRows}x{self.numCols}, nnz={self.values.size}, T={self.isTransposed})"


MLMatrix = Union[DenseMatrix, SparseMatrix]


@dataclass
class MatrixBlock:
    """M/matrix/MLMatrix.scala:1205."""
    rid: int
    cid: int
    matrix: MLMatrix


# ----------------------------------------------------------------------------------------------
# java.util.Random (JDK spec: 48-bit LCG) -- the rng behind DenseMatrix.rand / sprand
# ----------------------------------------------------------------------------------------------

_MULT = 0x5DEECE66D
_ADD = 0xB
_MASK = (1 << 48) - 1


class JavaRandom:
    def __init__(self, seed: int):
        self.seed = (seed ^ _MULT) & _MASK

    def next(self, bits: int) -> int:
        self.seed = (self.seed * _MULT + _ADD) & _MASK
        r = self.seed >> (48 - bits)
        if r >= 1 << (bits - 1) and bits == 32:
            r -= 1 << 32
        return r

    def nextDouble(self) -> float:
        return ((self.next(26) << 27) + self.next(27)) * (1.0 / (1 << 53))

    def nextInt(self, bound: int) -> int:
        r = self.next(31)
        m = bound - 1
        if (bound & m) == 0:
            return (bound * r) >> 31
        u = r
        while True:
            r = u % bound
            if u - r + m < (1 << 31):
                return r
            u = self.next(31)

    def next_doubles(self, n: int) -> np.ndarray:
        """n successive nextDouble() values, vectorised with LCG skip-ahead (exact)."""
        if n == 0:
            return np.zeros(0)
        # states s_1..s_2n: s_t = A^t s_0 + C_t.  Build by doubling.
        total = 2 * n
        a = np.empty(total, dtype=np.uint64)
        c = np.empty(total, dtype=np.uint64)
        a[0], c[0] = _MULT, _ADD
        filled = 1
        mask = np.uint64(_MASK)
        while filled < total:
            m = min(filled, total - filled)
            # compose step `filled` (a[filled-1], c[filled-1]) after steps 1..m
            af, cf = a[filled - 1], c[filled - 1]
            a[filled:filled + m] = (a[:m] * af) & mask
            c[filled:filled + m] = (c[:m] * af + cf) & mask
            filled += m
        s0 = np.uint64(self.seed)
        states = (a * s0 + c) & mask
        self.seed = int(states[-1])
        hi = (states[0::2] >> np.uint64(22)).astype(np.float64)  # next(26)
        lo = (states[1::2] >> np.uint64(21)).astype(np.float64)  # next(27)
        return (hi * float(1 << 27) + lo) * (1.0 / (1 << 53))


def sprand(numRows: int, numCols: int, density: float, rng: JavaRandom) -> SparseMatrix:
    """SparseMatrix.sprand, density < 0.34 branch (M/matrix/MLMatrix.scala:791-856).

    The reference collects entries in a scala mutable HashSet; its iteration order only
    affects which U(0,1) value lands on which coordinate, so the restatement orders
    coordinates column-major (the order fromCOO sorts them into, :730-760)."""
    require(numRows > 0, f"numRows must be greater than 0 but got {numRows}")
    require(numCols > 0, f"numCols must be greater than 0 but got {numCols}")
    require(0.0 <= density <= 1.0,
            f"density must be a double in the range 0.0 <= d <= 1.0. Currently, density: {density}")
    nnz = int(math.ceil(numRows * numCols * density))
    assert density < 0.34, "oracle restates only the draw-by-draw branch"
    entries = set()
    while len(entries) < nnz:
        entries.add((rng.nextInt(numRows), rng.nextInt(numCols)))
    coo = sorted(entries, key=lambda t: (t[1], t[0]))
    colPtrs = np.zeros(numCols + 1, dtype=np.int32)
    for _, j in coo:
        colPtrs[j + 1] += 1
    colPtrs = np.cumsum(colPtrs).astype(np.int32)
    rowIndices = np.array([i for i, _ in coo], dtype=np.int32)
    vals = rng.next_doubles(nnz)
    return SparseMatrix(numRows, numCols, colPtrs, rowIndices, vals)


# ----------------------------------------------------------------------------------------------
# Wire struct (M/util/MLMatrixSerializer.scala:26-69)
# ----------------------------------------------------------------------------------------------


def serialize(obj: MLMatrix) -> tuple:
    if isinstance(obj, SparseMatrix):
        return (0, obj.numRows, obj.numCols, obj.colPtrs.copy(), obj.rowIndices.copy(),
                obj.values.copy(), obj.isTransposed)
    return (1, obj.numRows, obj.numCols, None, None, obj.values.copy(), obj.isTransposed)


def deserialize(row: tuple) -> MLMatrix:
    require(len(row) == 7,
            f"MatrixUDT.deserialize given row with length {len(row)} but requires length == 7")
    tpe, numRows, numCols, colPtrs, rowIndices, values, isT = row
    if tpe == 0:
        return SparseMatrix(numRows, numCols, colPtrs, rowIndices, values, isT)
    return DenseMatrix(numRows, numCols, values, isT)


# ----------------------------------------------------------------------------------------------
# BLAS.gemm (M/matrix/BLAS.scala:301-458) and MLMatrix.multiply (M/matrix/MLMatrix.scala:100-104)
# ----------------------------------------------------------------------------------------------


def gemmddd(A: DenseMatrix, B: DenseMatrix) -> DenseMatrix:
    """C = zeros; dgemm(tA, tB, m, n, k, 1.0, A, lda, B, ldb, 0.0, C, ldc) (BLAS.scala:327-346)."""
    require(A.numCols == B.numRows,
            f"The columns of A don't match the rows of B. A: {A.numCols}, B: {B.numRows}")
    C = A.to_numpy() @ B.to_numpy()
    return DenseMatrix(A.numRows, B.numCols, np.ascontiguousarray(C.T).reshape(-1))


def gemmsdd_loops(A: SparseMatrix, B: DenseMatrix) -> DenseMatrix:
    """Literal restatement of the four loop nests of BLAS.gemmsdd (BLAS.scala:352-458) for
    alpha = 1, beta = 0 into a zeroed C.  Pure-Python loops: small cases only."""
    mA, nB, kA, kB = A.numRows, B.numCols, A.numCols, B.numRows
    require(kA == kB, f"The columns of A don't match the rows of B. A: {kA}, B: {kB}")
    C = np.zeros(mA * nB)
    Av, Ai, Ap = A.values, A.rowIndices, A.colPtrs
    for col in range(nB):
        Cstart = col * mA
        if A.isTransposed:            # CSR: row . column dot products (:375-413)
            for r in range(mA):
                s = 0.0
                for i in range(int(Ap[r]), int(Ap[r + 1])):
                    s += Av[i] * B.apply(int(Ai[i]), col)
                C[Cstart + r] = 0.0 * C[Cstart + r] + s * 1.0
        else:                         # CSC: scatter-AXPY (:414-456)
            for c in range(kA):
                bval = B.apply(c, col) * 1.0
                for i in range(int(Ap[c]), int(Ap[c + 1])):
                    C[Cstart + int(Ai[i])] += Av[i] * bval
    return DenseMatrix(mA, nB, C)


def gemmsdd(A: SparseMatrix, B: DenseMatrix) -> DenseMatrix:
    """Vectorised equivalent of :func:`gemmsdd_loops` (same sums, numpy order)."""
    require(A.numCols == B.numRows,
            f"The columns of A don't match the rows of B. A: {A.numCols}, B: {B.numRows}")
    import scipy.sparse as sp
    if A.isTransposed:
        S = sp.csr_matrix((A.values, A.rowIndices, A.colPtrs), shape=(A.numRows, A.numCols))
    else:
        S = sp.csc_matrix((A.values, A.rowIndices, A.colPtrs), shape=(A.numRows, A.numCols))
    C = np.asarray(S @ B.to_numpy())
    return DenseMatrix(A.numRows, B.numCols, np.ascontiguousarray(C.T).reshape(-1))


def multiplySparseMatDenseVec(spm: SparseMatrix, dv: DenseMatrix) -> DenseMatrix:
    """M/matrix/LocalMatrix.scala:856-887."""
    require(dv.numCols == 1, f"vector with more than 1 columns, dv.numCols = {dv.numCols}")
    require(spm.numCols == dv.numRows, "Sparse Mat-Vect dimensions do not match, "
            f"Mat.numCols = {spm.numCols}, Vec.numRows = {dv.numRows}")
    return DenseMatrix(spm.numRows, 1, spm.to_numpy() @ dv.to_numpy()[:, 0])


def multiplySparseSparse(ma: SparseMatrix, mb: SparseMatrix) -> MLMatrix:
    """LocalMatrix.multiplySparseSparse (M/matrix/LocalMatrix.scala:143-323).  The four loop nests (CSC x CSC :155-196,
    CSR x CSR :198-239, CSR x CSC :241-286, CSC x CSR :288-323) compute the same product over the STORED entries only and
    drop results that are exactly 0.0 (`!= 0.0`, so NaN is kept); they differ in the storage format of the result:
      CSC x CSC: CSC iff rows*cols > 2 nnz + (cols + 1), else that matrix .toDense
      CSR x CSR: CSR iff rows*cols > 2 nnz + (rows + 1), else .toDense
      CSR x CSC: always CSC (both branches construct the SparseMatrix, :280-285)
      CSC x CSR: dense iff rows*cols <= 2 nnz + cols, else DenseMatrix.toSparse (CSC)
    Summation order inside an entry follows scipy here, not the Scala loops (fp64 tolerance, not bit-exact)."""
    import scipy.sparse as sp
    require(ma.numCols == mb.numRows, "Matrix A.numCols must be equals to B.numRows, but found "
            f"A.numCols = {ma.numCols}, B.numRows = {mb.numRows}")

    def as_scipy(m: SparseMatrix):
        cls = sp.csr_matrix if m.isTransposed else sp.csc_matrix
        return cls((m.values, m.rowIndices, m.colPtrs), shape=(m.numRows, m.numCols))
    arr = np.asarray((as_scipy(ma) @ as_scipy(mb)).toarray(), dtype=np.float64)
    rows, cols = ma.numRows, mb.numCols
    nnz = int(np.count_nonzero(arr))
    dense = DenseMatrix(rows, cols, np.ascontiguousarray(arr.T).reshape(-1))
    csc = dense.toSparse()
    if not ma.isTransposed and not mb.isTransposed:
        return csc if rows * cols > 2 * nnz + cols + 1 else dense
    if ma.isTransposed and mb.isTransposed:
        csr = DenseMatrix(cols, rows, np.ascontiguousarray(arr).reshape(-1)).toSparse().transpose()
        return csr if rows * cols > 2 * nnz + rows + 1 else dense
    if ma.isTransposed and not mb.isTransposed:
        return csc
    return dense if rows * cols <= 2 * nnz + cols else csc


def matrixMultiplication(mat1: MLMatrix, mat2: MLMatrix) -> MLMatrix:
    """Type dispatch of M/matrix/LocalMatrix.scala:889-914."""
    d1, d2 = isinstance(mat1, DenseMatrix), isinstance(mat2, DenseMatrix)
    if d1 and d2:
        return gemmddd(mat1, mat2)
    if d1 and not d2:
        return gemmddd(mat1, mat2.toDense())                       # :892
    if not d1 and d2:
        if mat2.numCols == 1:
            return multiplySparseMatDenseVec(mat1, mat2)           # :894-896
        return gemmsdd(mat1, mat2)                                 # :898
    s1 = mat1.values.size * 1.0 / (mat1.numRows * mat1.numCols)
    s2 = mat2.values.size * 1.0 / (mat2.numRows * mat2.numCols)
    if s1 > 0.1:
        return gemmddd(mat1.toDense(), mat2.toDense())             # :903-904
    if s2 > 0.1:
        return gemmsdd(mat1, mat2.toDense())                       # :906-907
    return multiplySparseSparse(mat1, mat2)                        # :909-911


# ----------------------------------------------------------------------------------------------
# LocalMatrix element kernels (M/matrix/LocalMatrix.scala)
# ----------------------------------------------------------------------------------------------


def _sparse_or_dense_from_array(numRows: int, numCols: int, arr: np.ndarray) -> MLMatrix:
    """Output-format rule of the transposed sparse/sparse branches (LocalMatrix.scala:74-91,
    521-541): dense array, converted with toSparse iff rows*cols > 2*nnz + cols + 1."""
    nnz = int(np.count_nonzero(arr))
    c = DenseMatrix(numRows, numCols, arr)
    if numRows * numCols > nnz * 2 + numCols + 1:
        return c.toSparse()
    return c


def _native_sparse_rule(numRows: int, numCols: int, arr: np.ndarray) -> MLMatrix:
    """addSparseSparseNative / elementWiseOpSparseSparseNative tail (LocalMatrix.scala:133-138,
    596-601): CSC of the nonzeros, densified unless rows*cols > 2*nnz + (cols+1)."""
    s = DenseMatrix(numRows, numCols, arr).toSparse()
    if numRows * numCols > 2 * int(s.colPtrs[-1]) + s.colPtrs.size:
        return s
    return s.toDense()


def add(a: Optional[MLMatrix], b: Optional[MLMatrix]) -> Optional[MLMatrix]:
    """M/matrix/LocalMatrix.scala:34-54 (+ addDense :56-63, addDenseSparse :65-72,
    addSparseSparse :74-139).  Dense results are always column-major, isTransposed = false."""
    if a is None or b is None:
        return a if b is None else b
    require(a.numRows == b.numRows, "Matrix A and B must have the same number of rows. But found "
            f"A.numRows = {a.numRows}, B.numRows = {b.numRows}")
    require(a.numCols == b.numCols, "Matrix A and B must have the same number of cols. But found "
            f"A.numCols = {a.numCols}, B.numCols = {b.numCols}")
    arr = a.toArray() + b.toArray()
    if isinstance(a, SparseMatrix) and isinstance(b, SparseMatrix):
        if a.isTransposed or b.isTransposed:
            return _sparse_or_dense_from_array(a.numRows, a.numCols, arr)
        return _native_sparse_rule(a.numRows, a.numCols, arr)
    return DenseMatrix(a.numRows, a.numCols, arr)


def _elementwise(mat1: MLMatrix, mat2: MLMatrix, op: int, compat_bugs: bool) -> MLMatrix:
    require(mat1.numRows == mat2.numRows,
            f"mat1.numRows = {mat1.numRows}, mat2.numRows = {mat2.numRows}")
    require(mat1.numCols == mat2.numCols,
            f"mat1.numCols = {mat1.numCols}, mat2.numCols = {mat2.numCols}")
    x, y = mat1, mat2
    if isinstance(mat1, SparseMatrix) and isinstance(mat2, DenseMatrix) and compat_bugs:
        # defect B4: (Sparse, Dense) calls elementWiseOpDenseSparse(mb, ma, op): operands
        # swapped (LocalMatrix.scala:474,487).  Harmless for multiply, wrong for divide.
        x, y = mat2, mat1
    with np.errstate(divide="ignore", invalid="ignore"):
        arr = x.toArray() * y.toArray() if op == 0 else x.toArray() / y.toArray()
    if isinstance(mat1, SparseMatrix) and isinstance(mat2, SparseMatrix):
        if mat1.isTransposed or mat2.isTransposed:
            # `arr(i) != 0` counts NaN as nonzero (LocalMatrix.scala:533)
            return _sparse_or_dense_from_array(mat1.numRows, mat1.numCols, arr)
        return _native_sparse_rule(mat1.numRows, mat1.numCols, arr)
    return DenseMatrix(mat1.numRows, mat1.numCols, arr)


def elementWiseMultiply(mat1: MLMatrix, mat2: MLMatrix, compat_bugs: bool = True) -> MLMatrix:
    """M/matrix/LocalMatrix.scala:466-477, 493-519."""
    return _elementwise(mat1, mat2, 0, compat_bugs)


def elementWiseDivide(mat1: MLMatrix, mat2: MLMatrix, compat_bugs: bool = True) -> MLMatrix:
    """M/matrix/LocalMatrix.scala:479-490, 493-519."""
    return _elementwise(mat1, mat2, 1, compat_bugs)


def _map_values(mat: MLMatrix, f) -> MLMatrix:
    if isinstance(mat, DenseMatrix):
        return DenseMatrix(mat.numRows, mat.numCols, f(mat.values), mat.isTransposed)
    return SparseMatrix(mat.numRows, mat.numCols, mat.colPtrs, mat.rowIndices, f(mat.values),
                        mat.isTransposed)


def multiplyScalar(alpha: float, a: MLMatrix) -> MLMatrix:
    """M/matrix/LocalMatrix.scala:411-426 -- maps stored values, preserves isTransposed."""
    return _map_values(a, lambda v: alpha * v)


def addScalar(mat: MLMatrix, alpha: float) -> MLMatrix:
    """M/matrix/LocalMatrix.scala:965-980 -- stored values only (sparse zeros stay zero)."""
    return _map_values(mat, lambda v: v + alpha)


def matrixPow(mat: MLMatrix, p: float) -> MLMatrix:
    """M/matrix/LocalMatrix.scala:931-946 -- math.pow on stored values."""
    def f(v):
        with np.errstate(all="ignore"):
            return np.power(v, p)
    return _map_values(mat, f)


def rankOneAdd(mat1: MLMatrix, mat2: MLMatrix, mat3: MLMatrix, compat_bugs: bool = True) -> DenseMatrix:
    """M/matrix/LocalMatrix.scala:1075-1093.

    compat_bugs=True restates defect B3 literally: arr1 is never filled from mat1, so the result
    is x.y^T written at mat1's *storage* index k (and the result is flagged non-transposed even
    when mat1 is).  compat_bugs=False is the intended A + x.y^T (comment at
    M/plans/MatrixOperator.scala:151-152), column-major."""
    x = mat2.to_numpy()[:, 0]
    y = mat3.to_numpy()[:, 0]
    outer = np.outer(x[:mat1.numRows], y[:mat1.numCols])
    if not compat_bugs:
        res = mat1.to_numpy() + outer
        return DenseMatrix(mat1.numRows, mat1.numCols, np.ascontiguousarray(res.T).reshape(-1))
    arr = np.zeros(mat1.numRows * mat1.numCols)
    if not mat1.isTransposed:
        arr[:] = np.ascontiguousarray(outer.T).reshape(-1)      # k = i + numRows*j
    else:
        arr[:] = np.ascontiguousarray(outer).reshape(-1)        # k = j + numCols*i
    return DenseMatrix(mat1.numRows, mat1.numCols, arr)


# ----------------------------------------------------------------------------------------------
# Partitioners (M/partitioner/*.scala, M/execution/MatfastExecutionHelper.scala:46-62)
# ----------------------------------------------------------------------------------------------


def _java_round(x: float) -> int:
    return int(math.floor(x + 0.5))


def row_partition(i: int, j: int, partitions: int) -> int:
    """RowPartitioner.getPartition (M/partitioner/RowPartitioner.scala:32-38)."""
    return i % partitions


def column_partition(i: int, j: int, partitions: int) -> int:
    """ColumnPartitioner.getPartition (M/partitioner/ColumnPartitioner.scala:32-38)."""
    return j % partitions


def index_partition(i: int) -> int:
    """IndexPartitioner.getPartition (M/partitioner/IndexPartitioner.scala:29-34)."""
    return i


def gen_block_cyclic_partitioner(nrows: int, ncols: int, blkSize: int) -> Tuple[int, int, int, int]:
    """genBlockCyclicPartitioner (M/execution/MatfastExecutionHelper.scala:46-62)."""
    R = int(math.ceil(nrows * 1.0 / blkSize))
    C = int(math.ceil(ncols * 1.0 / blkSize))
    scale = 1.0 / math.sqrt(64)
    r = _java_round(max(scale * R, 1.0))
    c = _java_round(max(scale * C, 1.0))
    if r == 1 or c == 1:
        if r != 1:
            r = _java_round(max(r / 8.0, 1.0))
        if c != 1:
            c = _java_round(max(c / 8.0, 1.0))
    return (R, C, r, c)


class BlockCyclicPartitioner:
    """M/partitioner/BlockCyclicPartitioner.scala:31-62 (defect B2 restated literally)."""

    def __init__(self, ROW_BLKS: int, COL_BLKS: int, ROW_BLKS_PER_PARTITION: int,
                 COL_BLKS_PER_PARTITION: int):
        require(ROW_BLKS > 0, f"Number of row blocks should be larger than 0, but found {ROW_BLKS}")
        require(COL_BLKS > 0, f"Number of col blocks should be larger than 0, but found {COL_BLKS}")
        require(ROW_BLKS_PER_PARTITION > 0, "Number of row blocks per partition should be larger "
                f"than 0, but found {ROW_BLKS_PER_PARTITION}")
        require(COL_BLKS_PER_PARTITION > 0, "Number of col blocks per partition should be larger "
                f"than 0, but found {COL_BLKS_PER_PARTITION}")
        self.row_partition_num = int(math.ceil(ROW_BLKS * 1.0 / ROW_BLKS_PER_PARTITION))
        self.col_partition_num = int(math.ceil(COL_BLKS * 1.0 / COL_BLKS_PER_PARTITION))
        self.num_row_part = ROW_BLKS // self.row_partition_num
        self.num_col_part = COL_BLKS // self.col_partition_num
        self.numPartitions = self.row_partition_num * self.col_partition_num

    def getPartition(self, i: int, j: int) -> int:
        return ((i % self.num_row_part) * self.col_partition_num
                + (j % self.num_col_part)) % self.numPartitions


# ----------------------------------------------------------------------------------------------
# Physical operators (M/execution/MatfastExecution.scala, MatfastExecutionHelper.scala)
# A "dataset" is a dict {(rid, cid): MLMatrix}; absent keys are implicit zero blocks.
# ----------------------------------------------------------------------------------------------

BlockDict = Dict[Tuple[int, int], MLMatrix]


def to_block_dict(blocks: Iterable[MatrixBlock]) -> BlockDict:
    return {(b.rid, b.cid): b.matrix for b in blocks}


def matrix_multiply(left: BlockDict, leftRowNum: int, leftColNum: int, right: BlockDict,
                    rightRowNum: int, rightColNum: int, blkSize: int) -> BlockDict:
    """MatrixMatrixMultiplicationExecution.doExecute (MatfastExecution.scala:700-725) ->
    matrixMultiplyGeneral (MatfastExecutionHelper.scala:235-263) or the outer-product paths
    (:175-221).  Defect B1 (DuplicateLeft throws) is NOT restated: both outer-product variants
    return the mathematically intended cross product, as DuplicateRight does.
    The reduceByKey(add) order is arbitrary in Spark; the oracle sums in ascending k."""
    require(leftColNum == rightRowNum, "Matrix dimension not match, "
            f"leftColNum = {leftColNum}, rightRowNum = {rightRowNum}")
    leftColBlkNum = int(math.ceil(leftColNum * 1.0 / blkSize))
    rightRowBlkNum = int(math.ceil(rightRowNum * 1.0 / blkSize))
    out: BlockDict = {}
    if leftColBlkNum == 1 and rightRowBlkNum == 1:
        for (i, _), a in sorted(left.items()):
            for (_, j), b in sorted(right.items()):
                out[(i, j)] = matrixMultiplication(a, b)          # no reduce (:208-212)
        return out
    ks_left: Dict[int, List[Tuple[int, MLMatrix]]] = {}
    for (i, k), a in left.items():
        ks_left.setdefault(k, []).append((i, a))
    ks_right: Dict[int, List[Tuple[int, MLMatrix]]] = {}
    for (k, j), b in right.items():
        ks_right.setdefault(k, []).append((j, b))
    for k in sorted(set(ks_left) & set(ks_right)):               # join on k (:248)
        for i, a in ks_left[k]:
            for j, b in ks_right[k]:
                p = matrixMultiplication(a, b)                    # :250-254
                out[(i, j)] = p if (i, j) not in out else add(out[(i, j)], p)   # :255
    return out


def transpose(ds: BlockDict) -> BlockDict:
    """MatrixTransposeExecution (MatfastExecution.scala:215-236)."""
    return {(cid, rid): m.transpose() for (rid, cid), m in ds.items()}


def _check_same_dims(lr, lc, rr, rc):
    require(lr == rr, f"Row number not match, leftRowNum = {lr}, rightRowNum = {rr}")
    require(lc == rc, f"Col number not match, leftColNum = {lc}, rightColNum = {rc}")


def add_element(left: BlockDict, lr, lc, right: BlockDict, rr, rc, blkSize) -> BlockDict:
    """MatrixElementAddExecution (:583-607) + addWithPartitioner (helper :64-105): OUTER join;
    one-sided blocks pass through untouched (type and flags preserved)."""
    _check_same_dims(lr, lc, rr, rc)
    out: BlockDict = dict(left)
    for key, b in right.items():
        out[key] = add(out[key], b) if key in out else b
    return out


def multiply_element(left: BlockDict, lr, lc, right: BlockDict, rr, rc, blkSize,
                     compat_bugs: bool = True) -> BlockDict:
    """MatrixElementMultiplyExecution (:620-644) + multiplyWithPartitioner (helper :107-139): INNER join."""
    _check_same_dims(lr, lc, rr, rc)
    return {k: elementWiseMultiply(left[k], right[k], compat_bugs) for k in left if k in right}


def divide_element(left: BlockDict, lr, lc, right: BlockDict, rr, rc, blkSize,
                   compat_bugs: bool = True) -> BlockDict:
    """MatrixElementDivideExecution (:657-686) + divideWithPartitioner (helper :141-173): INNER join."""
    _check_same_dims(lr, lc, rr, rc)
    return {k: elementWiseDivide(left[k], right[k], compat_bugs) for k in left if k in right}


def add_scalar(ds: BlockDict, alpha: float) -> BlockDict:
    """MatrixScalarAddExecution (MatfastExecution.scala:465-486)."""
    return {k: addScalar(m, alpha) for k, m in ds.items()}


def multiply_scalar(ds: BlockDict, alpha: float) -> BlockDict:
    """MatrixScalarMultiplyExecution (MatfastExecution.scala:488-509)."""
    return {k: multiplyScalar(alpha, m) for k, m in ds.items()}


def power(ds: BlockDict, alpha: float) -> BlockDict:
    """MatrixPowerExecution (MatfastExecution.scala:511-532)."""
    return {k: matrixPow(m, alpha) for k, m in ds.items()}


def rank_one_update(left: BlockDict, lr, lc, right: BlockDict, rr, rc, blkSize,
                    compat_bugs: bool = True) -> BlockDict:
    """RankOneUpdateExecution (:728-747) + matrixRankOneUpdate (helper :265-285).

    compat_bugs=True keeps the reference's `require`s (which only admit 1-row matrices) and
    defect B3.  compat_bugs=False is the intended A + v.v^T for an n x n A and n x 1 v."""
    if compat_bugs:
        require(rr == 1, f"Vector column size is not 1, but #cols = {rr}")
        require(lr == rr, "Dimension not match for matrix addition, "
                f"A.nrows = {lr}, A.ncols = {lc}, B.nrows = {rr}, B.ncols = {rc}")
    else:
        require(rc == 1, f"Vector column size is not 1, but #cols = {rc}")
        require(lr == rr and lc == rr, "Dimension not match for matrix addition, "
                f"A.nrows = {lr}, A.ncols = {lc}, B.nrows = {rr}, B.ncols = {rc}")
    out: BlockDict = {}
    for (i, j), a in left.items():
        # x2.rid == i, x3.rid == j  (helper :271-275)
        xs = [m for (r, _), m in right.items() if r == i]
        ys = [m for (r, _), m in right.items() if r == j]
        for x in xs:
            for y in ys:
                out[(i, j)] = rankOneAdd(a, x, y, compat_bugs)
    return out


# ----------------------------------------------------------------------------------------------
# Aggregates (SURVEY.md section 8f-2): RowSum / ColumnSum / Sum / TraceDirectExecution
# (M/execution/MatfastExecution.scala:239-463).  literal=True restates the reference's index arithmetic
# as written (it is only correct for square dense blocks: non-square transposed blocks are mis-strided,
# CSR blocks are summed along the wrong axis, sparse ColumnSum has defect B5); literal=False is the
# mathematically intended reduction, which is what the GPU engine computes.
# ----------------------------------------------------------------------------------------------


def _row_sum_block(m: MLMatrix, literal: bool) -> DenseMatrix:
    if not literal:
        return DenseMatrix(m.numRows, 1, m.to_numpy().sum(axis=1))
    if isinstance(m, DenseMatrix):
        if not m.isTransposed:                                   # :254-261
            arr = np.zeros(m.numRows)
            np.add.at(arr, np.arange(m.values.size) % m.numRows, m.values)
            return DenseMatrix(m.numRows, 1, arr)
        n = m.numCols                                            # :262-271 ("column sum" branch)
        arr = np.zeros(n)
        for i in range(n):
            for j in range(m.numRows):
                arr[i] += m.values[i * m.numRows + j]
        return DenseMatrix(n, 1, arr)
    if not m.isTransposed:                                       # CSC :274-279
        arr = np.zeros(m.numRows)
        np.add.at(arr, m.rowIndices, m.values)
        return DenseMatrix(m.numRows, 1, arr)
    arr = np.zeros(m.numCols)                                    # CSR :280-287 (sums by column index)
    np.add.at(arr, m.rowIndices, m.values)
    return DenseMatrix(m.numCols, 1, arr)


def _col_sum_block(m: MLMatrix, literal: bool) -> DenseMatrix:
    if not literal:
        return DenseMatrix(1, m.numCols, m.to_numpy().sum(axis=0))
    if isinstance(m, DenseMatrix):
        if not m.isTransposed:                                   # :318-327
            n = m.numCols
            arr = np.array([m.values[i * m.numRows:(i + 1) * m.numRows].sum() for i in range(n)])
            return DenseMatrix(1, n, arr)
        mm = m.numRows                                           # :328-336
        arr = np.zeros(mm)
        np.add.at(arr, np.arange(m.values.size) % mm, m.values)
        return DenseMatrix(1, mm, arr)
    nlines = m.colPtrs.size - 1                                  # :338-357, defect B5: values(i + j)
    arr = np.zeros(nlines)
    for i in range(nlines):
        for j in range(int(m.colPtrs[i + 1] - m.colPtrs[i])):
            arr[i] += m.values[i + j]
    return DenseMatrix(1, nlines, arr)


def row_sum(ds: BlockDict, nrows: int, ncols: int, literal: bool = False) -> BlockDict:
    """Dataset.rowSum (M/Dataset.scala:63-66) -> RowSumDirectExecution: per-block sums, reduceByKey(add) on rid."""
    out: BlockDict = {}
    for (rid, _), m in sorted(ds.items()):
        v = _row_sum_block(m, literal)
        out[(rid, 0)] = v if (rid, 0) not in out else add(out[(rid, 0)], v)
    return out


def col_sum(ds: BlockDict, nrows: int, ncols: int, literal: bool = False) -> BlockDict:
    """Dataset.colSum (M/Dataset.scala:68-71) -> ColumnSumDirectExecution: reduceByKey(add) on cid."""
    out: BlockDict = {}
    for (_, cid), m in sorted(ds.items()):
        v = _col_sum_block(m, literal)
        out[(0, cid)] = v if (0, cid) not in out else add(out[(0, cid)], v)
    return out


def total_sum(ds: BlockDict, nrows: int, ncols: int) -> BlockDict:
    """Dataset.sum (M/Dataset.scala:73-76) -> SumDirectExecution (:377-391): values.sum per block (stored values)."""
    if not ds:
        return {}
    return {(0, 0): DenseMatrix(1, 1, [float(sum(float(m.values.sum()) for _, m in sorted(ds.items())))])}


def trace(ds: BlockDict, nrows: int, ncols: int) -> BlockDict:
    """Dataset.trace (M/Dataset.scala:78-82) -> TraceDirectExecution (:412-452): diagonal blocks only."""
    require(nrows == ncols, "Cannot perform trace() on a rectangle matrix")
    tr, seen = 0.0, False
    for (rid, cid), m in sorted(ds.items()):
        if rid != cid:
            continue
        seen = True
        if isinstance(m, DenseMatrix):
            require(m.numRows == m.numCols, f"block is not square, row_num={m.numRows}, col_num={m.numCols}")
        tr += float(np.trace(m.to_numpy()))
    return {(0, 0): DenseMatrix(1, 1, [tr])} if seen else {}


def project(ds: BlockDict, nrows: int, ncols: int, blkSize: int, rowOrCol: bool, index: int) -> BlockDict:
    """Dataset.project (M/Dataset.scala:38-47) -> Project{Row,Column}DirectExecution (MatfastExecution.scala:31-150),
    intended semantics: row `index` as 1 x cols blocks (0, cid) / column `index` as rows x 1 blocks (rid, 0)."""
    if rowOrCol:
        require(index < nrows, f"row index should be smaller than #rows, index={index}, #rows={nrows}")
    else:
        require(index < ncols, f"col index should be smaller than #cols, index={index}, #cols={ncols}")
    bid, off = index // blkSize, index % blkSize
    out: BlockDict = {}
    for (rid, cid), m in ds.items():
        a = m.to_numpy()
        if rowOrCol and rid == bid and off < m.numRows:
            out[(0, cid)] = DenseMatrix(1, m.numCols, a[off, :].copy())
        if not rowOrCol and cid == bid and off < m.numCols:
            out[(rid, 0)] = DenseMatrix(m.numRows, 1, a[:, off].copy())
    return out


def vec(ds: BlockDict, nrows: int, ncols: int, blkSize: int) -> BlockDict:
    """Dataset.vec (M/Dataset.scala:84-87) -> VectorizeExecution (MatfastExecution.scala:534-569), intended semantics:
    column t of block (i, j) -> rows x 1 block keyed ((j*blkSize + t) * ceil(nrows/blkSize) + i, 0).
    (Defect B6: the reference reads arr(t*numLocalCols + k) and keys with j*ROW_BLK_NUM*blkSize + t*ROW_BLK_NUM + i, which is
    the same key; only the stride differs and it is wrong for non-square blocks.)"""
    R = -(-nrows // blkSize)
    out: BlockDict = {}
    for (i, j), m in ds.items():
        a = m.to_numpy()
        for t in range(m.numCols):
            out[((j * blkSize + t) * R + i, 0)] = DenseMatrix(m.numRows, 1, a[:, t].copy())
    return out


def selection(ds: BlockDict, nrows: int, ncols: int, blkSize: int, rowIdx: int, colIdx: int) -> BlockDict:
    """Dataset.selection (M/Dataset.scala:49-55) -> SelectDirectExecution (MatfastExecution.scala:152-213)."""
    require(rowIdx < nrows, f"row index should be smaller than #rows, rid={rowIdx}, #rows={nrows}")
    require(colIdx < ncols, f"col index should be smaller than #cols, cid={colIdx}, #cols={ncols}")
    key = (rowIdx // blkSize, colIdx // blkSize)
    if key not in ds:
        return {}
    return {(0, 0): DenseMatrix(1, 1, [ds[key].apply(rowIdx % blkSize, colIdx % blkSize)])}


# ----------------------------------------------------------------------------------------------
# helpers for tests / bench
# ----------------------------------------------------------------------------------------------


def assemble(ds: BlockDict, nrows: int, ncols: int, blkSize: int) -> np.ndarray:
    """Dense nrows x ncols array from a block dict (absent blocks are zeros)."""
    out = np.zeros((nrows, ncols))
    for (i, j), m in ds.items():
        out[i * blkSize:i * blkSize + m.numRows, j * blkSize:j * blkSize + m.numCols] = m.to_numpy()
    return out


def rand_dense_dataset(nrows: int, ncols: int, blkSize: int, seed0: int,
                       transposed_mask=None) -> BlockDict:
    """Synthetic input of SURVEY.md section 8d: every block present, U(0,1) from
    java.util.Random(seed0 + rid*ncolblks + cid) in storage order."""
    nbr = -(-nrows // blkSize)
    nbc = -(-ncols // blkSize)
    ds: BlockDict = {}
    for i in range(nbr):
        for j in range(nbc):
            r = min(blkSize, nrows - i * blkSize)
            c = min(blkSize, ncols - j * blkSize)
            m = DenseMatrix.rand(r, c, JavaRandom(seed0 + i * nbc + j))
            if transposed_mask is not None and transposed_mask(i, j):
                m = DenseMatrix(r, c, m.values, True)
            ds[(i, j)] = m
    return ds

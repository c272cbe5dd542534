"""The reference's element-wise joins with a sparse side, restated loop for loop with numpy.

`sparse_sparse` is LocalMatrix.addSparseSparse / elementWiseOpSparseSparse (M/matrix/LocalMatrix.scala:74-139, :521-602) of one
block pair and `dense_sparse` is addDenseSparse / elementWiseOpDenseSparse (:65-72, :507-519).  op is 'add', 'mul' or 'div'; every
operation is one rounded IEEE operation (numpy float64 scalars and arrays never fuse).

  1. both operands CSC: the native loops.  coltmp starts at 0.0 and each stored entry is added in storage order, so repeats are
     summed and a stored -0.0 becomes +0.0; add runs ONE sum per row over A's entries then B's, multiply / divide take op(a, b)
     of the two columns.  Entries != 0.0 are kept, rows ascending; the result is that CSC iff rows*cols > 2 nnz + cols + 1, else its
     toDense (+0.0 wherever nothing is kept).
  2. either operand CSR: op over the toArray images (the last stored entry of a position wins, sign kept), the same rule, and
     toSparse (CSC) of the array or the array itself.
  3. dense (+) sparse: op over the toArray images, always dense.

A result is (fmt, values, ptr, idx): fmt 'dense' or 'csc'; values the m x n array (dense) or the stored values (csc) with their
column pointers and row indices.
"""
import numpy as np

DENSE, CSC = "dense", "csc"
OPS = {"add": np.add, "mul": np.multiply, "div": np.divide}


def _entries(s):
    """(row, col, value) of every stored entry of a sparse block, in foreachActive order (MLMatrix.scala:637-663)."""
    ptr, idx, val = np.asarray(s.colPtrs), np.asarray(s.rowIndices), np.asarray(s.values, dtype=np.float64)
    for line in range(len(ptr) - 1):
        for e in range(ptr[line], ptr[line + 1]):
            yield (line, int(idx[e]), val[e]) if s.isTransposed else (int(idx[e]), line, val[e])


def to_array(s):
    """SparseMatrix.toArray as an m x n array: the last stored entry of a position wins."""
    a = np.zeros((s.numRows, s.numCols))
    for r, c, v in _entries(s):
        a[r, c] = v
    return a


def dense_array(d):
    """DenseMatrix.toArray as an m x n array (isTransposed honoured)."""
    v = np.asarray(d.values, dtype=np.float64)
    return v.reshape(d.numRows, d.numCols) if d.isTransposed else v.reshape(d.numCols, d.numRows).T


def to_sparse(arr):
    """DenseMatrix.toSparse (MLMatrix.scala:353-374): the entries != 0.0 (NaN kept, -0.0 dropped), column by column."""
    ptr, idx, val = [0], [], []
    for c in range(arr.shape[1]):
        nz = np.nonzero(arr[:, c] != 0.0)[0]
        idx.extend(nz.tolist())
        val.extend(arr[nz, c].tolist())
        ptr.append(len(idx))
    return np.asarray(ptr, np.int32), np.asarray(idx, np.int32), np.asarray(val, np.float64)


def _rule(m, n, nnz):
    return m * n > 2 * nnz + n + 1


def sparse_sparse(op, a, b):
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        return _sparse_sparse(op, a, b)


def _sparse_sparse(op, a, b):
    m, n = a.numRows, a.numCols
    f = OPS[op]
    if a.isTransposed or b.isTransposed:          # case 2: the toArray branch
        arr = f(to_array(a), to_array(b))
        ptr, idx, val = to_sparse(arr)
        return (CSC, val, ptr, idx) if _rule(m, n, len(val)) else (DENSE, arr, None, None)
    ap, ai, av = np.asarray(a.colPtrs), np.asarray(a.rowIndices), np.asarray(a.values, dtype=np.float64)
    bp, bi, bv = np.asarray(b.colPtrs), np.asarray(b.rowIndices), np.asarray(b.values, dtype=np.float64)
    ptr, idx, val = [0], [], []
    for jc in range(n):                           # case 1: the native loops
        tmp1 = np.zeros(m)
        for ia in range(ap[jc], ap[jc + 1]):
            tmp1[ai[ia]] += av[ia]
        if op == "add":
            for ib in range(bp[jc], bp[jc + 1]):
                tmp1[bi[ib]] += bv[ib]
        else:
            tmp2 = np.zeros(m)
            for ib in range(bp[jc], bp[jc + 1]):
                tmp2[bi[ib]] += bv[ib]
            tmp1 = f(tmp1, tmp2)
        nz = np.nonzero(tmp1 != 0.0)[0]
        idx.extend(nz.tolist())
        val.extend(tmp1[nz].tolist())
        ptr.append(len(idx))
    ptr, idx, val = np.asarray(ptr, np.int32), np.asarray(idx, np.int32), np.asarray(val, np.float64)
    if _rule(m, n, len(val)):
        return CSC, val, ptr, idx
    arr = np.zeros((m, n))                        # toDense of the CSC
    for c in range(n):
        arr[idx[ptr[c]:ptr[c + 1]], c] = val[ptr[c]:ptr[c + 1]]
    return DENSE, arr, None, None


def dense_sparse(op, d, s, sparse_left):
    """Case 3: op(d, s), or op(s, d) when sparse_left (a (Sparse, Dense) pair without defect B4's swap)."""
    x, y = dense_array(d), to_array(s)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        arr = OPS[op](y, x) if sparse_left else OPS[op](x, y)
    return DENSE, arr, None, None


def bits(v):
    """float64 values as int64 bits, every NaN mapped to one pattern (payloads may differ)."""
    v = np.array(v, dtype=np.float64, copy=True).reshape(-1)
    v[np.isnan(v)] = np.nan
    return v.view(np.int64)


def assert_block(got, want, key=None):
    """A block the engine returned (DenseMatrix / SparseMatrix) against a result of this module, bit for bit."""
    fmt, v, ptr, idx = want
    sparse = type(got).__name__ == "SparseMatrix"
    assert sparse == (fmt == CSC), (key, type(got).__name__, fmt)
    assert not got.isTransposed, key
    if fmt == DENSE:
        assert (got.numRows, got.numCols) == v.shape, key
        assert np.array_equal(bits(got.values), bits(v.T.reshape(-1))), key
    else:
        assert np.array_equal(np.asarray(got.colPtrs), ptr), key
        assert np.array_equal(np.asarray(got.rowIndices), idx), key
        assert np.array_equal(bits(got.values), bits(v)), key

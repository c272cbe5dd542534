"""The reference's sparse x sparse block product and its partial sums, restated loop for loop with numpy.

`pair_product` is LocalMatrix.multiplySparseSparse (LocalMatrix.scala:143-323) for one block pair and `add` is LocalMatrix.add
(:30-139) of two partials; `multiply` chains them over the k-blocks in ascending k, as the engine does for output blocks whose
partials are all low-density sparse x sparse.  Every product and every sum is rounded on its own: each step is one
`acc[idx] += vals * b`, which numpy evaluates as a rounded product followed by a rounded sum (it never fuses them).

A result is (fmt, values): fmt 'dense', 'csc' or 'csr', values the m x n array of the block (absent entries 0.0).  A sparse
result's stored entries are exactly its values != 0.0 (NaN included), in ascending index order.
"""
import numpy as np

DENSE, CSC, CSR = "dense", "csc", "csr"


def _dense_and_mask(s):
    """The m x n values and stored-entry mask of a sparse block (CSC, or CSR when isTransposed)."""
    m, n = s.numRows, s.numCols
    d, mask = np.zeros((m, n)), np.zeros((m, n), dtype=bool)
    ptr, idx, val = np.asarray(s.colPtrs), np.asarray(s.rowIndices), np.asarray(s.values)
    line = np.repeat(np.arange(len(ptr) - 1), np.diff(ptr))
    r, c = (line, idx) if s.isTransposed else (idx, line)
    d[r, c] = val
    mask[r, c] = True
    return d, mask


def _walk_lines(ptr):
    """For the stored positions t = 0, 1, ...: (the lines holding a t-th entry, the index of that entry)."""
    ptr = np.asarray(ptr)
    lens = np.diff(ptr)
    for t in range(int(lens.max()) if lens.size else 0):
        lines = np.nonzero(lens > t)[0]
        yield lines, ptr[lines] + t


def pair_product(a, b):
    """multiplySparseSparse of two sparse blocks: (fmt, values).  Inf x 0 gives NaN as in the JVM, without numpy's warning."""
    with np.errstate(invalid="ignore", over="ignore"):
        return _pair_product(a, b)


def _pair_product(a, b):
    m, n = a.numRows, b.numCols
    c = np.zeros((m, n))
    if not a.isTransposed and not b.isTransposed:      # multiplyCSC_CSC: column j of B in stored order
        ad, am = _dense_and_mask(a)
        bi, bv = np.asarray(b.rowIndices), np.asarray(b.values)
        for cols, pos in _walk_lines(b.colPtrs):
            k, alpha = bi[pos], bv[pos]
            c[:, cols] += np.where(am[:, k], ad[:, k] * alpha, 0.0)
    elif a.isTransposed:                                # multiplyCSR_CSR / multiplyCSR_CSC: row i of A in stored order
        bd, bm = _dense_and_mask(b)
        ai, av = np.asarray(a.rowIndices), np.asarray(a.values)
        for rows, pos in _walk_lines(a.colPtrs):
            k, alpha = ai[pos], av[pos]
            c[rows, :] += np.where(bm[k, :], alpha[:, None] * bd[k, :], 0.0)
    else:                                               # multiplyCSC_CSR: outer products in ascending k
        ap, ai, av = np.asarray(a.colPtrs), np.asarray(a.rowIndices), np.asarray(a.values)
        bp, bi, bv = np.asarray(b.colPtrs), np.asarray(b.rowIndices), np.asarray(b.values)
        for k in range(a.numCols):
            r, x = ai[ap[k]:ap[k + 1]], av[ap[k]:ap[k + 1]]
            q, y = bi[bp[k]:bp[k + 1]], bv[bp[k]:bp[k + 1]]
            if r.size and q.size:
                c[np.ix_(r, q)] += np.outer(x, y)
    nnz = int(np.count_nonzero(c != 0.0))
    cells = m * n
    if not a.isTransposed and not b.isTransposed:
        fmt = CSC if cells > 2 * nnz + n + 1 else DENSE
    elif a.isTransposed and b.isTransposed:
        fmt = CSR if cells > 2 * nnz + m + 1 else DENSE
    elif a.isTransposed:
        fmt = CSC
    else:
        fmt = DENSE if cells <= 2 * nnz + n else CSC
    return fmt, c


def add(s, p):
    """LocalMatrix.add of two partials: dense if either is dense, else CSC iff rows*cols > 2 nnz + cols + 1."""
    (fs, vs), (fp, vp) = s, p
    v = vs + vp
    if fs == DENSE or fp == DENSE:
        return DENSE, v
    m, n = v.shape
    return (CSC if m * n > 2 * int(np.count_nonzero(v != 0.0)) + n + 1 else DENSE), v


def multiply(A, B):
    """The chain outputs of A x B (block dicts {(i, j): sparse block}, every pair sparse x sparse): {(i, j): (fmt, values)},
    partials added in ascending k."""
    out = {}
    for (i, k) in sorted(A):
        for (k2, j) in sorted(B):
            if k2 != k:
                continue
            a, b = A[(i, k)], B[(k, j)]
            for blk in (a, b):  # LocalMatrix.scala:900-911 sends only pairs of density <= 0.1 to multiplySparseSparse
                assert len(blk.values) <= 0.1 * blk.numRows * blk.numCols, "not a low-density sparse x sparse pair"
            p = pair_product(a, b)
            out[(i, j)] = add(out[(i, j)], p) if (i, j) in out else p
    return out


def dump(res):
    """(kind, isTransposed, rows, cols, values as int64 bits, colPtrs, rowIndices), the layout the GPU tests compare."""
    fmt, v = res
    m, n = v.shape
    if fmt == DENSE:
        vals = np.where(v == 0.0, 0.0, v).T.reshape(-1)
        return ("dense", False, m, n, vals.view(np.int64).copy(), None, None)
    w = v if fmt == CSC else v.T
    ptr, idx, val = [0], [], []
    for c in range(w.shape[1]):
        nz = np.nonzero(w[:, c] != 0.0)[0]
        idx.append(nz)
        val.append(w[nz, c])
        ptr.append(ptr[-1] + nz.size)
    idx = np.concatenate(idx).astype(np.int32) if idx else np.zeros(0, np.int32)
    val = np.concatenate(val).astype(np.float64) if val else np.zeros(0)
    return ("sparse", fmt == CSR, m, n, val.view(np.int64).copy(), np.asarray(ptr, dtype=np.int32), idx)

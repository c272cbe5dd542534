"""The matrix x vector products C = A x and C = x A of DESIGN section 4.5.5, restated with numpy.

Every product and every add is rounded on its own (numpy float64 operations do not contract), so these functions give the bits
the route must give:
  - a pair's partial starts at +0.0 and adds its terms one by one:
      A x, dense A:  c ascending;                   A x, CSR A: each row in storage order;
      A x, CSC A:    columns ascending, each in storage order (LocalMatrix.multiplySparseMatDenseVec), repeats each count;
      x A, dense A:  r ascending;
      x A, sparse A: the terms of the dense image in storage order: only the last stored entry of a position counts, and the
                     partial is NaN where a non-finite x[r] meets a position (r, j) that is not stored;
  - the partials of an output block are combined in ascending k: S = p_k0, then S + p_k1, and so on.
Blocks are any objects with numRows, numCols, values, isTransposed (and colPtrs, rowIndices when sparse)."""
import numpy as np


def is_sparse(b):
    return hasattr(b, "colPtrs")


def dense_array(b):
    v = np.asarray(b.values, dtype=np.float64)
    if b.isTransposed:
        return v.reshape(b.numRows, b.numCols)
    return v.reshape(b.numCols, b.numRows).T


def entries(b):
    """(line, index, value) of every stored entry in storage order; lines are rows of a CSR block, columns of a CSC one."""
    ptr = np.asarray(b.colPtrs, dtype=np.int64)
    line = np.repeat(np.arange(ptr.size - 1), np.diff(ptr))
    return line, np.asarray(b.rowIndices, dtype=np.int64), np.asarray(b.values, dtype=np.float64)


def last_stored(line, idx):
    """Mask of the entries no later entry of the same position overwrites."""
    keep = np.ones(line.size, dtype=bool)
    seen = set()
    for e in range(line.size - 1, -1, -1):
        key = (int(line[e]), int(idx[e]))
        if key in seen:
            keep[e] = False
        seen.add(key)
    return keep


def partial(a, x, xa):
    """p_k of one pair: matrix block a, vector x (a.numCols values for A x, a.numRows for x A)."""
    x = np.asarray(x, dtype=np.float64).reshape(-1)
    n = a.numCols if xa else a.numRows
    p = np.zeros(n)
    if not is_sparse(a):
        M = dense_array(a)
        M = M.T if xa else M
        with np.errstate(invalid="ignore", over="ignore"):
            for c in range(M.shape[1]):
                p = p + M[:, c] * x[c]
        return p
    line, idx, val = entries(a)
    row, col = (line, idx) if a.isTransposed else (idx, line)
    out, w = (col, row) if xa else (row, col)
    if xa:
        keep = last_stored(line, idx)
        out, w, val = out[keep], w[keep], val[keep]
    with np.errstate(invalid="ignore", over="ignore"):
        np.add.at(p, out, val * x[w])       # in storage order, one rounded add per term
    if xa:
        for r in np.flatnonzero(~np.isfinite(x)):
            stored = np.zeros(n, dtype=bool)
            stored[out[w == r]] = True
            p[~stored] = np.nan
    return p


def combine(parts):
    S = parts[0].copy()
    with np.errstate(invalid="ignore", over="ignore"):
        for p in parts[1:]:
            S = S + p
    return S


def product(A, X, xa):
    """C = A x (xa False: A the left blocks, X the k x 1 right blocks) or C = x A (xa True: X the 1 x k left blocks, A the right
    blocks), as {(rid, cid): values} with the output blocks of the join on k (ascending k)."""
    pairs = {}
    if xa:
        for (_, k), xb in X.items():
            for (k2, j), a in A.items():
                if k2 == k:
                    pairs.setdefault((0, j), []).append((k, a, xb))
    else:
        for (i, k), a in A.items():
            for (k2, _), xb in X.items():
                if k2 == k:
                    pairs.setdefault((i, 0), []).append((k, a, xb))
    return {key: combine([partial(a, xb.values, xa) for _, a, xb in sorted(ps, key=lambda t: t[0])])
            for key, ps in pairs.items()}

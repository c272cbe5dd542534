"""The aggregates and slicing of sparse blocks on their stored entries (DESIGN section 4.5.4), restated with numpy.

  1. rowSum / colSum: a sparse block's partial at output index t is ((0.0 + v1) + v2) + ... over its stored entries at index t in
     storage order (the reference's per-entry loops, MatfastExecution.scala:273-287, :337-356 with colPtrs(i) + j).  Repeats each
     count; explicit zeros, -0.0 and non-finite values take part.  The partials of one output line are combined in ascending block
     index: S = ((0.0 + p_b0) + p_b1) + ....  A line that also has dense blocks adds S to their sum (fp64 atomics, any order).
  2. trace: ((0.0 + v1) + v2) + ... over the stored entries with row == column, in storage order, per diagonal block; the blocks
     combined as in 1.
  3. project / selection: the value at a position is its LAST stored entry in storage order (toArray / foreachActive,
     MLMatrix.scala:637-663), 0.0 where nothing is stored, sign and NaN kept.

np.add.at is unbuffered and applies its updates one by one in the order of its index array, each a rounded fp64 add; with zeros
as the start it is exactly the running sums of rule 1 (test_sparse_agg_ref_cpu.py checks this against plain Python loops).
"""
import numpy as np


def is_sparse(m):
    return type(m).__name__ == "SparseMatrix"


def coords(s):
    """(rows, cols, values) of every stored entry of a sparse block, in storage order."""
    ptr = np.asarray(s.colPtrs, dtype=np.int64)
    idx = np.asarray(s.rowIndices, dtype=np.int64)[ptr[0]:ptr[-1]]
    val = np.asarray(s.values, dtype=np.float64)[ptr[0]:ptr[-1]]
    line = np.repeat(np.arange(ptr.size - 1), np.diff(ptr))
    return (line, idx, val) if s.isTransposed else (idx, line, val)


def partial(op, s):
    """Rule 1 / 2 for one sparse block: 'row' -> [numRows], 'col' -> [numCols], 'trace' -> [1]."""
    r, c, v = coords(s)
    if op == "row":
        out, at = np.zeros(s.numRows), r
    elif op == "col":
        out, at = np.zeros(s.numCols), c
    else:
        keep = r == c
        out, at, v = np.zeros(1), np.zeros(int(keep.sum()), dtype=np.int64), v[keep]
    with np.errstate(invalid="ignore", over="ignore"):
        np.add.at(out, at, v)
    return out


def combine(parts):
    """S = ((0.0 + p0) + p1) + ..., element by element."""
    s = np.zeros_like(parts[0])
    with np.errstate(invalid="ignore", over="ignore"):
        for p in parts:
            s = s + p
    return s


def _key(op, rid, cid):
    return (rid, 0) if op == "row" else (0, cid) if op == "col" else (0, 0)


def aggregate(op, ds):
    """{output key: (S of the sparse blocks or None, [dense blocks of the line])} for op in 'row', 'col', 'trace'.  A key whose
    dense list is empty has exactly S as its output."""
    out = {}
    for (rid, cid), m in sorted(ds.items()):
        if op == "trace" and rid != cid:
            continue
        parts, dense = out.setdefault(_key(op, rid, cid), ([], []))
        (parts if is_sparse(m) else dense).append(m)
    res = {}
    for key, (parts, dense) in out.items():
        S = combine([partial(op, m) for m in parts]) if parts else None
        res[key] = (S, dense)
    return res


def terms(op, ds, key, t):
    """The values that add up to output element t of `key` (every stored sparse entry at t and every dense element at t)."""
    vals = []
    for (rid, cid), m in sorted(ds.items()):
        if (op == "trace" and rid != cid) or _key(op, rid, cid) != key:
            continue
        if is_sparse(m):
            r, c, v = coords(m)
            sel = (r == c) if op == "trace" else (r == t) if op == "row" else (c == t)
            vals.append(v[sel])
        else:
            a = m.to_numpy()
            vals.append(np.diag(a) if op == "trace" else a[t, :] if op == "row" else a[:, t])
    return np.concatenate(vals) if vals else np.zeros(0)


def _last(keys, v, n):
    """out[k] = the last v with that key (0.0 where none), out of n."""
    out = np.zeros(n)
    if keys.size:
        u, first = np.unique(keys[::-1], return_index=True)
        out[u] = v[::-1][first]
    return out


def line_of(m, take_row, offset):
    """Row (take_row) or column `offset` of a block: a sparse block's last stored entries, a dense block's elements."""
    if not is_sparse(m):
        a = m.to_numpy()
        return (a[offset, :] if take_row else a[:, offset]).copy()
    r, c, v = coords(m)
    if take_row:
        sel = r == offset
        return _last(c[sel], v[sel], m.numCols)
    sel = c == offset
    return _last(r[sel], v[sel], m.numRows)


def entry_of(m, i, j):
    """Entry (i, j) of a block: the last stored entry there, or 0.0."""
    if not is_sparse(m):
        return float(m.to_numpy()[i, j])
    r, c, v = coords(m)
    hit = np.flatnonzero((r == i) & (c == j))
    return float(v[hit[-1]]) if hit.size else 0.0


def project(ds, blk, take_row, index):
    """{key: values} of Dataset.project: row `index` as 1 x cols blocks (0, cid), column `index` as rows x 1 blocks (rid, 0)."""
    bid, off = index // blk, index % blk
    out = {}
    for (rid, cid), m in ds.items():
        if take_row and rid == bid and off < m.numRows:
            out[(0, cid)] = line_of(m, True, off)
        if not take_row and cid == bid and off < m.numCols:
            out[(rid, 0)] = line_of(m, False, off)
    return out


def selection(ds, blk, i, j):
    key = (i // blk, j // blk)
    m = ds.get(key)
    if m is None or i % blk >= m.numRows or j % blk >= m.numCols:
        return {}
    return {(0, 0): np.array([entry_of(m, i % blk, j % blk)])}


def bits(v):
    """float64 values as int64 bits, every NaN mapped to one pattern (payloads may differ)."""
    v = np.array(v, dtype=np.float64, copy=True).reshape(-1)
    v[np.isnan(v)] = np.nan
    return v.view(np.int64)


def sum_bound(x):
    """|computed - exact| of a sum of the values x in any order with fp64 atomics: 1.01 (t + 2) 2^-53 sum |x| for t terms."""
    x = np.asarray(x, dtype=np.float64)
    return 1.01 * (x.size + 2) * 2.0 ** -53 * float(np.abs(x).sum())


"""Exact reference for block products with sparse operands, and the error bound of any summation order of the terms they form.

BLAS.gemmsdd (M/matrix/BLAS.scala:352-458) and LocalMatrix.multiplySparseMatDenseVec (LocalMatrix.scala:856-887) multiply each
STORED entry of a sparse left block -- explicit zeros and duplicate indices included -- with the B element it faces; no other
element of B is read.  So entry (i, j) of a product is a sum over exactly those terms (plus all of k for a dense left block,
LocalMatrix.scala:891-892, or a sparse one above 10 % density next to a sparse right block, :903-904), added over the k-blocks.
Its exact value comes from tests/exact_ref.exact_dot of the term vectors, and the bound counts the terms of that entry, not
the full inner dimension: a dropped, doubled or misplaced entry moves the result by a whole term, far outside it."""
import os
import re
from fractions import Fraction

import numpy as np

from oracle import matrel_oracle as O
from tests.exact_ref import ROOT, exact_dot

TINY = 2.0 ** -1074


def _sparse(b):
    return isinstance(b, O.SparseMatrix)


def _density(b):
    return b.values.size / (b.numRows * b.numCols)


def _all_of_k(a, b):
    """True when the pair multiplies dense images (every k is a term), False when it walks the stored entries of a."""
    return not _sparse(a) or (_sparse(b) and _density(a) > 0.1)


def _row_entries(a, r):
    """(column indices, values) of the stored entries of row r of a sparse block, in storage order."""
    if a.isTransposed:
        lo, hi = int(a.colPtrs[r]), int(a.colPtrs[r + 1])
        return a.rowIndices[lo:hi].astype(np.int64), a.values[lo:hi]
    major = np.repeat(np.arange(a.numCols), np.diff(a.colPtrs))
    sel = a.rowIndices == r
    return major[sel], a.values[sel]


def _dense_image(b):
    return b.to_numpy()


def _abs_image(a):
    """|a| with duplicate stored entries added (each one is its own term)."""
    if not _sparse(a):
        return np.abs(a.to_numpy())
    out = np.zeros((a.numRows, a.numCols))
    major = np.repeat(np.arange(a.colPtrs.size - 1), np.diff(a.colPtrs))
    rows, cols = (major, a.rowIndices) if a.isTransposed else (a.rowIndices, major)
    np.add.at(out, (rows, cols), np.abs(a.values))
    return out


def _stored_image(a):
    """Number of terms each element of a forms (stored entries of a sparse block, every element of a dense one)."""
    if not _sparse(a):
        return np.ones((a.numRows, a.numCols))
    out = np.zeros((a.numRows, a.numCols))
    major = np.repeat(np.arange(a.colPtrs.size - 1), np.diff(a.colPtrs))
    rows, cols = (major, a.rowIndices) if a.isTransposed else (a.rowIndices, major)
    np.add.at(out, (rows, cols), 1.0)
    return out


def _row_counts(a):
    """Number of terms of each row of a (stored entries of a sparse block, all of k for a dense one)."""
    if a.isTransposed:
        return np.diff(a.colPtrs).astype(np.int64)
    return np.bincount(a.rowIndices, minlength=a.numRows).astype(np.int64)


def entry_terms(A_blocks, B_blocks, k, blk, i, j):
    """(a values, b values) of every term the reference forms for C[i, j], k-block by k-block."""
    bi, ii, bj, jj = i // blk, i % blk, j // blk, j % blk
    av, bv = [], []
    for kb in range(-(-k // blk)):
        a, b = A_blocks.get((bi, kb)), B_blocks.get((kb, bj))
        if a is None or b is None:
            continue
        col = _dense_image(b)[:, jj]
        if _all_of_k(a, b):
            av.append(_dense_image(a)[ii, :])
            bv.append(col)
        else:
            idx, vals = _row_entries(a, ii)
            av.append(vals)
            bv.append(col[idx])
    if not av:
        return np.zeros(0), np.zeros(0)
    return np.concatenate(av), np.concatenate(bv)


def exact_sparse_entries(A_blocks, B_blocks, n, k, m, blk, positions):
    """Exact C[i, j] for each (i, j) of positions, as Fractions, over the terms the reference forms (finite data only)."""
    assert all(0 <= i < n and 0 <= j < m for i, j in positions)
    return [exact_dot(*entry_terms(A_blocks, B_blocks, k, blk, i, j)) for i, j in positions]


def sparse_sum_bound(A_blocks, B_blocks, n, k, m, blk):
    """Element-wise bound of |got - exact| for ANY order of the t_ij terms of C[i, j] (FMA chains, per-pair sums, atomics):
    1.01 (t_ij + 2) 2^-53 sum|terms| + (t_ij + 4) 2^-1074.  The + 2 covers the final C + sum of a partial product and the
    accumulation onto a dense partial."""
    S = np.zeros((n, m))
    T = np.zeros((n, m), dtype=np.int64)
    with np.errstate(over="ignore"):
        for (bi, kb), a in A_blocks.items():
            for bj in range(-(-m // blk)):
                b = B_blocks.get((kb, bj))
                if b is None:
                    continue
                rs, cs = slice(bi * blk, bi * blk + a.numRows), slice(bj * blk, bj * blk + b.numCols)
                Bd = _dense_image(b)
                fin = np.isfinite(Bd)
                absA = _abs_image(a) if not _all_of_k(a, b) else np.abs(_dense_image(a))
                # a non-finite B element only counts where a term faces it (an unreferenced row of B is never read)
                hit = ((_stored_image(a) if not _all_of_k(a, b) else np.ones(absA.shape)) @ (~fin)) > 0
                S[rs, cs] += np.where(hit, np.inf, absA @ np.where(fin, np.abs(Bd), 0.0))
                T[rs, cs] += (np.full(a.numRows, a.numCols) if _all_of_k(a, b) else _row_counts(a))[:, None]
        return 1.01 * (T + 2) * 2.0 ** -53 * S + (T + 4) * TINY


def nonfinite_class(A_blocks, B_blocks, n, k, m, blk, positions):
    """IEEE outcome ('nan', '+inf', '-inf' or 'finite') of each C[i, j], from its terms alone.  Valid for data built so that no
    finite partial sum overflows in an order-dependent way: then a NaN term, or +inf next to -inf, gives NaN; else an infinite
    term decides the sign.  The deterministic kernels multiply-add with FMA, which keeps an overflowing product unrounded: next
    to an infinity of the opposite sign it gives that infinity, not NaN, so cases must not mix the two."""
    out = []
    with np.errstate(over="ignore", invalid="ignore"):
        for i, j in positions:
            a, b = entry_terms(A_blocks, B_blocks, k, blk, i, j)
            p = a * b
            pos, neg = bool(np.any(p == np.inf)), bool(np.any(p == -np.inf))
            out.append("nan" if np.any(np.isnan(p)) or (pos and neg) else "+inf" if pos else "-inf" if neg else "finite")
    return out


def within(got, exact, bound):
    """|got - exact| <= bound for an fp64 result and an exact Fraction (finite data)."""
    return bool(np.isfinite(got)) and abs(Fraction(float(got)) - exact) <= Fraction(float(bound))


def classify(x):
    return "nan" if np.isnan(x) else "+inf" if x == np.inf else "-inf" if x == -np.inf else "finite"


def reference_product(A_blocks, B_blocks, n, k, m, blk):
    """The whole product with scipy.sparse for sparse left blocks (stored entries only, as gemmsdd) and numpy for dense pairs."""
    import scipy.sparse as sp
    C = np.zeros((n, m))
    with np.errstate(over="ignore", invalid="ignore"):
        for (bi, kb), a in A_blocks.items():
            for bj in range(-(-m // blk)):
                b = B_blocks.get((kb, bj))
                if b is None:
                    continue
                Bd = _dense_image(b)
                if _all_of_k(a, b):
                    P = _dense_image(a) @ Bd
                else:
                    fmt = sp.csr_matrix if a.isTransposed else sp.csc_matrix
                    P = np.asarray(fmt((a.values, a.rowIndices, a.colPtrs), shape=(a.numRows, a.numCols)) @ Bd)
                C[bi * blk:bi * blk + a.numRows, bj * blk:bj * blk + b.numCols] += P
    return C


# ---- the segment geometry of the pipelined kernel, read from its source so that the capacity tests follow the code
_CSRC = os.path.join(ROOT, "matrel_b200", "csrc")


def segment_params():
    """TM (rows of a strip), TN (columns of a tile), KC (k extent of a chunk), E_CAP (entries of a segment held in shared
    memory) and NCW (consumer warps) of spmm2_kernel."""
    src = open(os.path.join(_CSRC, "spmm.cu")).read()
    hdr = open(os.path.join(_CSRC, "kernels.h")).read()

    def const(name):
        v = re.search(r"constexpr int %s = (\w+);" % name, src).group(1)
        return int(v) if v.isdigit() else int(re.search(r"\b%s = (\d+)" % v, hdr).group(1))
    return {name: const(name) for name in ("TM", "TN", "KC", "E_CAP", "NCW")}

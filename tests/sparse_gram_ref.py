"""The host side of the sparse Gram route (DESIGN section 4.1.2), restated on top of tests/jvm_sparse_ref.py.

A Gram product L x R has R(k, j) = L(j, k)^T over the same arrays.  The route runs the chains of the blocks on and above the
diagonal, and of the non-square blocks below it; it derives the formats of the others, and of the diagonal blocks, from counts:
  - a triangular (diagonal) chain counts, per level, nnz(P_l) and the nnz(S_l) steps over rows r <= c, and the same two counts on
    the diagonal; the full block's counts are 2 upper - diagonal (P_l and S_l of a diagonal block are symmetric);
  - a square block (j, i) below the diagonal replays the format rules with its own pairs' layouts (L(j, k).isT, R(k, i).isT) and
    the counts of its mirror (i, j): nnz(P_l) and nnz(S_l) do not change under transposition.
"""
import numpy as np

from tests import jvm_sparse_ref as J


def transpose(blocks):
    """The blocks of the transposed dataset, over the same arrays (what A.t() makes)."""
    return {(j, i): type(m)(m.numCols, m.numRows, m.colPtrs, m.rowIndices, m.values, not m.isTransposed)
            for (i, j), m in blocks.items()}


def levels(L, R, i, j):
    """The pairs of output block (i, j) in ascending k."""
    return [(L[(i2, k)], R[(k, j)]) for (i2, k) in sorted(L) if i2 == i and (k, j) in R]


def chain_counts(L, R, i, j, region="all"):
    """Per level: (nnz(P_l), nnz(S_l) - nnz(S_l-1)) of output block (i, j) over its rows r <= c ("upper"), its diagonal ("diag")
    or all of it."""
    cp, cs = [], []
    S, prev = None, 0
    for a, b in levels(L, R, i, j):
        _, P = J.pair_product(a, b)
        S = P if S is None else S + P
        m, n = P.shape
        mask = {"all": np.ones((m, n), bool), "upper": np.triu(np.ones((m, n), bool)), "diag": np.eye(m, n, dtype=bool)}[region]
        now = int(np.count_nonzero(S[mask] != 0.0))
        cp.append(int(np.count_nonzero(P[mask] != 0.0)))
        cs.append(now - prev)
        prev = now
    return cp, cs


def full_counts(up, dg):
    """The counts of a symmetric block from those of its upper triangle and its diagonal."""
    return [2 * u - d for u, d in zip(up, dg)]


def chain_format(layouts, m, n, cp, cs):
    """The reference's format rules (partial formats, then the sum rule) replayed from per-level counts."""
    fmt, s_nnz = None, 0
    for (aT, bT), p, s in zip(layouts, cp, cs):
        s_nnz += s
        cells = m * n
        if not aT and not bT:
            pf = J.CSC if cells > 2 * p + n + 1 else J.DENSE
        elif aT and bT:
            pf = J.CSR if cells > 2 * p + m + 1 else J.DENSE
        elif aT:
            pf = J.CSC
        else:
            pf = J.DENSE if cells <= 2 * p + n else J.CSC
        if fmt is None:
            fmt = pf
        elif fmt == J.DENSE or pf == J.DENSE:
            fmt = J.DENSE
        else:
            fmt = J.CSC if cells > 2 * s_nnz + n + 1 else J.DENSE
    return fmt


def layouts_of(L, R, i, j):
    return [(a.isTransposed, b.isTransposed) for a, b in levels(L, R, i, j)]


def gram_formats(L, R, algebra=full_counts, mirror_layouts=True):
    """{(i, j): format} of every output block as the route decides it.  algebra / mirror_layouts=False plant defects: another
    full-count rule, and a mirrored block replayed with its mirror's layouts instead of its own."""
    out = {}
    ids = {(i, j) for (i, k) in L for (k2, j) in R if k2 == k}
    for (i, j) in ids:
        a, b = levels(L, R, i, j)[0]
        m, n = a.numRows, b.numCols
        if i == j:
            up, dg = chain_counts(L, R, i, i, "upper"), chain_counts(L, R, i, i, "diag")
            cp, cs = algebra(up[0], dg[0]), algebra(up[1], dg[1])
            out[(i, j)] = chain_format(layouts_of(L, R, i, j), m, n, cp, cs)
        elif i > j and m == n:
            cp, cs = chain_counts(L, R, j, i)
            lay = layouts_of(L, R, i, j) if mirror_layouts else layouts_of(L, R, j, i)
            out[(i, j)] = chain_format(lay, m, n, cp, cs)
        else:
            out[(i, j)] = chain_format(layouts_of(L, R, i, j), m, n, *chain_counts(L, R, i, j))
    return out

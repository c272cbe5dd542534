"""C = A X and C = X A for a thin side X of up to 8 columns (A X) or rows (X A), DESIGN section 4.5.5, restated column by column.

Column j of C (row j for X A) is the width-1 product of tests/matvec_ref.py on column j of X (row j), built from its `partial` and
`combine`, so these are the bits of t separate matrix x vector products.  Output blocks may have any width, so a thin side cut into
several block columns (blk < t) is covered as well."""
import numpy as np

from tests import matvec_ref as R


def vectors(xb, xa):
    """The vectors of a thin block: its columns for A X, its rows for X A."""
    a = R.dense_array(xb)
    return [a[j, :] for j in range(a.shape[0])] if xa else [a[:, j] for j in range(a.shape[1])]


def product(A, X, xa):
    """C = A X (xa False: A the left blocks, X the right blocks) or C = X A (xa True: X the left blocks, A the right blocks), as
    {(rid, cid): 2-D array} over the output blocks of the join on k, partials in ascending k."""
    pairs = {}
    if xa:
        for (r, k), xb in X.items():
            for (k2, c), a in A.items():
                if k2 == k:
                    pairs.setdefault((r, c), []).append((k, a, xb))
    else:
        for (r, k), a in A.items():
            for (k2, c), xb in X.items():
                if k2 == k:
                    pairs.setdefault((r, c), []).append((k, a, xb))
    out = {}
    for key, ps in pairs.items():
        ps = sorted(ps, key=lambda t: t[0])
        width = len(vectors(ps[0][2], xa))
        cols = [R.combine([R.partial(a, vectors(xb, xa)[j], xa) for _, a, xb in ps]) for j in range(width)]
        out[key] = np.stack(cols, axis=0 if xa else 1)
    return out

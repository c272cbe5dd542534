"""CPU checks of the sparse Gram route's host algebra (tests/sparse_gram_ref.py) against the JVM loops of the full product:
the full counts of a triangular chain, the counts a mirrored block shares with its mirror, and every block's format."""
import numpy as np
import pytest
import scipy.sparse as sp

from oracle import matrel_oracle as O
from tests import jvm_sparse_ref as J
from tests import sparse_gram_ref as G


def _block(a, csr):
    t = sp.csr_matrix(a) if csr else sp.csc_matrix(a)
    t.sort_indices()
    return O.SparseMatrix(a.shape[0], a.shape[1], t.indptr, t.indices, t.data, csr)


def _rand(rng, m, n, density):
    return np.where(rng.random((m, n)) < density, rng.uniform(0.5, 1.5, (m, n)) * rng.choice([-1.0, 1.0], (m, n)), 0.0)


def _low_density(rng, m, n, density):
    """A random block at most 0.1 dense (drawn again until it is: the chains take no denser block)."""
    while True:
        a = _rand(rng, m, n, density)
        if np.count_nonzero(a) <= 0.1 * m * n:
            return a


def _dataset(rng, M, N, blk, density, csr):
    return {(i, j): _block(_low_density(rng, min(blk, M - i * blk), min(blk, N - j * blk), density), csr(i, j))
            for i in range(-(-M // blk)) for j in range(-(-N // blk))}


def _special(rng):
    """Stored zeros, a product that cancels to 0.0, Inf and NaN (A A^T, blk 12)."""
    A = _dataset(rng, 30, 36, 12, 0.06, lambda i, j: (i + j) % 2 == 0)
    a = _rand(rng, 12, 12, 0.06)
    a[0, :] = 0.0
    a[2, 3], a[5, 7] = np.inf, np.nan
    b = _block(a, False)
    vals = b.values.copy()
    vals[np.nonzero(np.isfinite(vals))[0][:2]] = 0.0
    A[(0, 0)] = O.SparseMatrix(12, 12, b.colPtrs, b.rowIndices, vals, False)
    z = np.zeros((12, 12))
    A[(1, 0)] = _block(z, True)
    for k, sgn in ((1, 1.0), (2, -1.0)):
        x, y = z.copy(), z.copy()
        x[0, 0], y[0, 0] = 1.0, sgn
        A[(0, k)], A[(1, k)] = _block(x, k == 1), _block(y, False)
    return A


LAYOUTS = {"csc": lambda i, j: False, "csr": lambda i, j: True, "mixed": lambda i, j: (3 * i + j) % 2 == 0}


def cases():
    out = []
    for layout, f in LAYOUTS.items():
        for density in (0.01, 0.05, 0.09):              # sparse-ending chains, and chains that flip to dense mid-way
            for kind in ("AAt", "AtA"):
                out.append((f"{layout}-{density}-{kind}", kind, (100, 90, 40, density, f)))
    out.append(("ragged-outer-mixed", "AAt", (100, 30, 40, 0.08, LAYOUTS["mixed"])))
    return out


def _operands(A, kind):
    return (A, G.transpose(A)) if kind == "AAt" else (G.transpose(A), A)


def _build(spec, seed):
    M, N, blk, density, f = spec
    return _dataset(np.random.default_rng(seed), M, N, blk, density, f)


def check(L, R, **plant):
    want = J.multiply(L, R)
    got = G.gram_formats(L, R, **plant)
    assert got == {k: v[0] for k, v in want.items()}
    algebra = plant.get("algebra", G.full_counts)
    for (i, j) in want:
        if i == j:
            up, dg = G.chain_counts(L, R, i, i, "upper"), G.chain_counts(L, R, i, i, "diag")
            assert (algebra(up[0], dg[0]), algebra(up[1], dg[1])) == G.chain_counts(L, R, i, i)
        elif i > j:
            assert G.chain_counts(L, R, i, j) == G.chain_counts(L, R, j, i)


@pytest.mark.parametrize("name,kind,spec", cases(), ids=[c[0] for c in cases()])
def test_formats_and_counts(name, kind, spec):
    check(*_operands(_build(spec, len(name)), kind))


def test_stored_zeros_cancellation_and_nonfinite():
    A = _special(np.random.default_rng(3))
    L, R = _operands(A, "AAt")
    check(L, R)
    C = J.multiply(L, R)
    assert C[(0, 1)][1][0, 0] == 0.0 and np.isnan(C[(0, 0)][1]).any()


def test_formats_cover_every_kind():
    """The cases above end dense, CSC and CSR (a single-level CSR x CSR mirror of a CSC x CSC block)."""
    seen = set()
    for name, kind, spec in cases():
        seen |= set(G.gram_formats(*_operands(_build(spec, len(name)), kind)).values())
    assert seen == {J.DENSE, J.CSC, J.CSR}


def test_a_wrong_full_count_is_caught():
    L, R = _operands(_build((100, 90, 40, 0.05, LAYOUTS["csc"]), 1), "AAt")
    with pytest.raises(AssertionError):
        check(L, R, algebra=lambda up, dg: [2 * u for u in up])


def test_a_wrong_layout_pairing_is_caught():
    """One k-block, block row 0 CSR and the others CSC: block (0, j) is CSR x CSR (a CSR result), its mirror CSC x CSC."""
    kind, spec = "AAt", (100, 30, 40, 0.02, lambda i, j: i == 0)
    L, R = _operands(_build(spec, 5), kind)
    check(L, R)
    with pytest.raises(AssertionError):
        check(L, R, mirror_layouts=False)

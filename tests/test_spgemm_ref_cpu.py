"""The restated sparse x sparse loops (tests/jvm_sparse_ref.py), without a GPU: values against scipy, storage formats against the
oracle's block multiply."""
import numpy as np
import pytest
import scipy.sparse as sp

from oracle import matrel_oracle as O
from tests import jvm_sparse_ref as J


def sparse_block(a, csr):
    """O.SparseMatrix of the dense array a: CSC, or CSR (isTransposed) when csr."""
    if csr:
        t = sp.csr_matrix(a)
        t.sort_indices()
        return O.SparseMatrix(a.shape[0], a.shape[1], t.indptr, t.indices, t.data, True)
    t = sp.csc_matrix(a)
    t.sort_indices()
    return O.SparseMatrix(a.shape[0], a.shape[1], t.indptr, t.indices, t.data, False)


def random_sparse(rng, m, n, density):
    return np.where(rng.random((m, n)) < density, rng.uniform(-1, 1, (m, n)), 0.0)


@pytest.mark.parametrize("fa,fb", [(False, False), (True, True), (True, False), (False, True)])
@pytest.mark.parametrize("density", [0.01, 0.08])
def test_pair_product_matches_scipy_and_the_oracle(fa, fb, density):
    rng = np.random.default_rng(int(density * 100) + 2 * fa + fb)
    a, b = random_sparse(rng, 70, 50, density), random_sparse(rng, 50, 61, density)
    A, B = sparse_block(a, fa), sparse_block(b, fb)
    fmt, v = J.pair_product(A, B)
    np.testing.assert_allclose(v, (sp.csr_matrix(a) @ sp.csr_matrix(b)).toarray(), rtol=1e-13, atol=1e-15)
    want = O.matrix_multiply({(0, 0): A}, 70, 50, {(0, 0): B}, 50, 61, 100)[(0, 0)]
    kind, isT, m, n, bits, ptr, idx = J.dump((fmt, v))
    assert (kind == "sparse") == isinstance(want, O.SparseMatrix)
    assert (isT, m, n) == (want.isTransposed, want.numRows, want.numCols)
    if kind == "sparse":
        assert ptr.tolist() == want.colPtrs.tolist() and idx.tolist() == want.rowIndices.tolist()
    np.testing.assert_allclose(bits.view(np.float64), want.values, rtol=1e-13, atol=1e-15)


@pytest.mark.parametrize("fmt", ["csc", "csr", "mix"])
def test_chains_match_scipy_and_the_oracle(fmt):
    rng = np.random.default_rng({"csc": 1, "csr": 2, "mix": 3}[fmt])
    n, blk = 4 * 30 - 7, 30
    nb = -(-n // blk)
    for density in (0.01, 0.05):
        full = {}
        dA, dB = {}, {}
        for name, d in (("A", dA), ("B", dB)):
            for i in range(nb):
                for j in range(nb):
                    r, c = min(blk, n - i * blk), min(blk, n - j * blk)
                    csr = fmt == "csr" or (fmt == "mix" and rng.random() < 0.5)
                    d[(i, j)] = sparse_block(random_sparse(rng, r, c, density), csr)
            full[name] = O.assemble(d, n, n, blk)
        got = J.multiply(dA, dB)
        want = O.matrix_multiply(dA, n, n, dB, n, n, blk)
        assert sorted(got) == sorted(want)
        dense = np.zeros((n, n))
        for key, res in got.items():
            kind, isT, *_ , ptr, idx = J.dump(res)
            w = want[key]
            assert (kind == "sparse") == isinstance(w, O.SparseMatrix) and isT == w.isTransposed, key
            if kind == "sparse":
                assert ptr.tolist() == w.colPtrs.tolist() and idx.tolist() == w.rowIndices.tolist()
            i, j = key
            dense[i * blk:i * blk + res[1].shape[0], j * blk:j * blk + res[1].shape[1]] = res[1]
        np.testing.assert_allclose(dense, full["A"] @ full["B"], rtol=1e-12, atol=1e-14)


def test_zeros_are_dropped_and_nan_kept():
    """A product that cancels to exactly 0.0 leaves no entry; a stored zero times Inf is NaN and stays."""
    a = np.array([[1.0, 1.0], [0.0, 2.0]])
    b = np.array([[3.0, 0.0], [-1.5, 0.0]])
    fmt, v = J.pair_product(sparse_block(a, False), sparse_block(b, False))
    assert v[1, 0] == -3.0 and v[0, 0] == 1.5
    A = O.SparseMatrix(2, 1, [0, 2], [0, 1], [0.0, 1.0])        # an explicitly stored zero
    B = O.SparseMatrix(1, 1, [0, 1], [0], [np.inf])
    fmt, v = J.pair_product(A, B)
    assert np.isnan(v[0, 0]) and v[1, 0] == np.inf
    c = np.array([[1.0], [1.0]])
    d = np.array([[1.0, -1.0]])
    fmt, v = J.add(J.pair_product(sparse_block(c, False), sparse_block(d, False)),
                   J.pair_product(sparse_block(c, False), sparse_block(-d, False)))
    assert np.count_nonzero(v) == 0

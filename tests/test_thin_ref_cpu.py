"""CPU checks of tests/thin_ref.py: the golden 3-column sparse products, the oracle on integer data (where every order gives the
same bits), and hand-worked X S cases whose non-finite values sit in one column of X only."""
import json
import os

import numpy as np
import pytest

from oracle import matrel_oracle as O
from tests import matvec_ref as R
from tests import thin_ref as T

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def dense(a, rowmajor=False):
    a = np.asarray(a, dtype=np.float64)
    return O.DenseMatrix(a.shape[0], a.shape[1], np.ascontiguousarray(a if rowmajor else a.T).reshape(-1), rowmajor)


def csc(rows, cols, ptr, idx, val):
    return O.SparseMatrix(rows, cols, np.asarray(ptr, np.int32), np.asarray(idx, np.int32), np.asarray(val, np.float64), False)


def csr(rows, cols, ptr, idx, val):
    return O.SparseMatrix(rows, cols, np.asarray(ptr, np.int32), np.asarray(idx, np.int32), np.asarray(val, np.float64), True)


@pytest.mark.parametrize("rowmajor", [False, True])
def test_golden_three_column_products(rowmajor):
    g = json.load(open(os.path.join(GOLDEN, "test_sparse.json")))
    s1, s2 = O.SparseMatrix(**g["spmat1"]), O.SparseMatrix(**g["spmat2"])
    S1, S2 = np.asarray(g["S1_full"]), np.asarray(g["S2_full"])
    ex = g["expected"]
    for name, a, x in (("S1_times_S2", s1, S2), ("S1_times_S2t", s1, S2.T), ("S2_times_S2t", s2, S2.T)):
        got = T.product({(0, 0): a}, {(0, 0): dense(x, rowmajor)}, False)[(0, 0)]
        assert got.tolist() == ex[name], name
    # X S: S1 S2 with S1 as the thin (3-row) side and S2 sparse; S2 S2^T with S2 dense on the left
    assert T.product({(0, 0): s2}, {(0, 0): dense(S1, rowmajor)}, True)[(0, 0)].tolist() == ex["S1_times_S2"]
    assert T.product({(0, 0): s2.transpose()}, {(0, 0): dense(S2, rowmajor)}, True)[(0, 0)].tolist() == ex["S2_times_S2t"]


@pytest.mark.parametrize("xa", [False, True])
@pytest.mark.parametrize("kind", ["dense_col", "dense_row", "csc", "csr"])
@pytest.mark.parametrize("t,blk", [(3, 32), (8, 32), (5, 2)])
def test_integer_data_matches_the_oracle(kind, xa, t, blk):
    rng = np.random.default_rng(len(kind) + xa + 10 * t)
    n, k = (70, 90) if blk > 8 else (7, 9)
    rows, cols = (k, n) if xa else (n, k)
    A = {}
    for i in range(-(-rows // blk)):
        for j in range(-(-cols // blk)):
            r, c = min(blk, rows - i * blk), min(blk, cols - j * blk)
            a = np.where(rng.random((r, c)) < 0.3, rng.integers(-9, 10, (r, c)), 0).astype(np.float64)
            A[(i, j)] = {"dense_col": lambda: dense(a), "dense_row": lambda: dense(a, True),
                         "csc": lambda: dense(a).toSparse(), "csr": lambda: dense(a.T).toSparse().transpose()}[kind]()
    x = rng.integers(-9, 10, (t, k) if xa else (k, t)).astype(np.float64)
    xr, xc = x.shape
    X = {(i, j): dense(x[i * blk:(i + 1) * blk, j * blk:(j + 1) * blk], rowmajor=(i + j) % 2 == 1)
         for i in range(-(-xr // blk)) for j in range(-(-xc // blk))}
    want = O.matrix_multiply(X, t, k, A, k, n, blk) if xa else O.matrix_multiply(A, n, k, X, k, t, blk)
    got = T.product(A, X, xa)
    assert sorted(got) == sorted(want)
    for key in want:
        assert np.array_equal(got[key], O.assemble({(0, 0): want[key]}, want[key].numRows, want[key].numCols, blk * 1000)), key


def test_columns_are_the_width_one_products():
    rng = np.random.default_rng(5)
    a = csr(6, 5, [0, 2, 2, 5, 6, 6, 8], [4, 1, 0, 3, 0, 2, 1, 1], rng.uniform(-1, 1, 8))
    x = rng.uniform(-1, 1, (5, 3))
    got = T.product({(0, 0): a}, {(0, 0): dense(x, True)}, False)[(0, 0)]
    for j in range(3):
        assert np.array_equal(got[:, j], R.partial(a, x[:, j], False))


def test_non_finite_x_in_one_column_only():
    # CSC 3 x 2: column 0 stores rows 0 and 2, column 1 stores row 1
    a = csc(3, 2, [0, 2, 3], [0, 2, 1], [1.0, 7.0, 2.0])
    X = np.ones((2, 3))
    X[0, 1] = np.inf                                 # row 0 of X meets (1, 0), not stored: NaN there; (1, 1) stored: inf
    got = T.product({(0, 0): a}, {(0, 0): dense(X)}, True)[(0, 0)]
    assert got[1].tolist() == [8.0, 2.0]             # row 1 of X is untouched
    assert np.isnan(got[0, 0]) and got[0, 1] == np.inf
    X[1, 0] = np.nan                                 # row 1: NaN at r = 0, stored in column 0 only
    got = T.product({(0, 0): a}, {(0, 0): dense(X)}, True)[(0, 0)]
    assert np.isnan(got[1]).all() and np.isnan(got[0, 0]) and got[0, 1] == np.inf
    # the same matrix as CSR: A X never reads an X(c, j) that no stored entry references
    b = csr(2, 3, [0, 2, 3], [0, 2, 1], [1.0, 7.0, 2.0])
    Y = np.ones((3, 2))
    Y[1, 1] = np.inf
    got = T.product({(0, 0): b}, {(0, 0): dense(Y)}, False)[(0, 0)]
    assert got[:, 0].tolist() == [8.0, 2.0] and got[0, 1] == 8.0 and got[1, 1] == np.inf


def test_repeats_unsorted_lines_and_negative_zero():
    # CSC 3 x 3, column 0: rows 2, 0, 2 (a repeat, unsorted); column 1: row 1 holds -0.0
    a = csc(3, 3, [0, 3, 4, 4], [2, 0, 2, 1], [1.0, 2.0, 3.0, -0.0])
    X = np.array([[0.5, 1.0], [4.0, -1.0], [np.inf, 2.0]])
    got = T.product({(0, 0): a}, {(0, 0): dense(X)}, False)[(0, 0)]
    assert got[:, 0].tolist() == [1.0, 0.0, 2.0] and not np.signbit(got[1, 0])     # repeats each count; +0.0 + -0.0
    assert got[:, 1].tolist() == [2.0, 0.0, 4.0]
    # X A: the last stored entry of a repeated position counts
    got = T.product({(0, 0): a}, {(0, 0): dense(X.T, True)}, True)[(0, 0)]
    assert got[1].tolist() == [1.0 * 2.0 + 2.0 * 3.0, 0.0, 0.0]                # (2, 0) holds 3.0, not 1.0

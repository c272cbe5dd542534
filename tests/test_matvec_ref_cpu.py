"""CPU checks of tests/matvec_ref.py: the golden sparse x vector row, the oracle on integer data (where every order gives the same
bits), and hand-worked repeats, unsorted lines, -0.0 and non-finite values."""
import json
import os

import numpy as np
import pytest

from oracle import matrel_oracle as O
from tests import matvec_ref as R

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def csc(rows, cols, ptr, idx, val):
    return O.SparseMatrix(rows, cols, np.asarray(ptr, np.int32), np.asarray(idx, np.int32), np.asarray(val, np.float64), False)


def csr(rows, cols, ptr, idx, val):
    return O.SparseMatrix(rows, cols, np.asarray(ptr, np.int32), np.asarray(idx, np.int32), np.asarray(val, np.float64), True)


def dense(a, rowmajor=False):
    a = np.asarray(a, dtype=np.float64)
    vals = np.ascontiguousarray(a if rowmajor else a.T).reshape(-1)
    return O.DenseMatrix(a.shape[0], a.shape[1], vals, rowmajor)


def test_golden_sparse_times_vector():
    g = json.load(open(os.path.join(GOLDEN, "test_sparse.json")))
    s1 = O.SparseMatrix(**g["spmat1"])
    got = R.partial(s1, np.asarray(g["denV"], dtype=np.float64), False)
    assert got.tolist() == g["expected"]["S1_times_v"]


@pytest.mark.parametrize("xa", [False, True])
@pytest.mark.parametrize("kind", ["dense_col", "dense_row", "csc", "csr"])
def test_integer_data_matches_the_oracle(kind, xa):
    rng = np.random.default_rng(len(kind) + xa)
    n, k, blk = 70, 90, 32
    A = {}
    for i in range(-(-(k if xa else n) // blk)):
        for j in range(-(-(n if xa else k) // blk)):
            r = min(blk, (k if xa else n) - i * blk)
            c = min(blk, (n if xa else k) - j * blk)
            a = np.where(rng.random((r, c)) < 0.3, rng.integers(-9, 10, (r, c)), 0).astype(np.float64)
            A[(i, j)] = {"dense_col": lambda: dense(a), "dense_row": lambda: dense(a, True),
                         "csc": lambda: dense(a).toSparse(), "csr": lambda: dense(a.T).toSparse().transpose()}[kind]()
    x = rng.integers(-9, 10, k).astype(np.float64)
    if xa:
        X = {(0, j): O.DenseMatrix(1, min(blk, k - j * blk), x[j * blk:(j + 1) * blk]) for j in range(-(-k // blk))}
        want = O.matrix_multiply(X, 1, k, A, k, n, blk)
    else:
        X = {(i, 0): O.DenseMatrix(min(blk, k - i * blk), 1, x[i * blk:(i + 1) * blk]) for i in range(-(-k // blk))}
        want = O.matrix_multiply(A, n, k, X, k, 1, blk)
    got = R.product(A, X, xa)
    assert sorted(got) == sorted(want)
    for key in want:
        assert np.array_equal(got[key], np.asarray(want[key].values)), key


def test_hand_worked_csc_times_vector():
    # column 0: rows 2, 0, 2 (a repeat, unsorted); column 1: row 1 holds -0.0; column 2: nothing
    a = csc(3, 3, [0, 3, 4, 4], [2, 0, 2, 1], [1.0, 2.0, 3.0, -0.0])
    x = np.array([0.5, 4.0, np.inf])                       # x[2] is referenced by no stored entry
    p = R.partial(a, x, False)
    assert p.tolist() == [1.0, 0.0, 2.0]                   # row 2: 0.5 + 1.5 (repeats each count); row 1: +0.0 + -0.0 = +0.0
    assert np.signbit(p[1]) == False
    assert R.partial(a, np.array([np.nan, 1.0, 1.0]), False)[1] == 0.0


def test_hand_worked_csr_times_vector():
    a = csr(2, 3, [0, 3, 4], [2, 0, 2, 1], [1.0, 2.0, 3.0, 0.0])
    p = R.partial(a, np.array([1.0, np.inf, 2.0]), False)
    assert p[0] == 1.0 * 2.0 + 2.0 * 1.0 + 3.0 * 2.0      # unsorted row with a repeat, in storage order
    assert np.isnan(p[1])                                  # a stored 0.0 facing inf
    p = R.partial(a, np.array([1e308, 1.0, 1e308]), False)
    assert p[0] == np.inf                                  # 1e308 + 2e308 + 3e308 overflows


def test_hand_worked_vector_times_sparse():
    # CSC 3 x 2: column 0 stores row 0 twice (the last value, 5.0, counts) and row 2; column 1 stores row 1
    a = csc(3, 2, [0, 3, 4], [0, 2, 0, 1], [1.0, 7.0, 5.0, 2.0])
    p = R.partial(a, np.array([1.0, 1.0, 1.0]), True)
    assert p.tolist() == [7.0 + 5.0, 2.0]
    p = R.partial(a, np.array([1.0, np.inf, 1.0]), True)  # x[1] meets (1, 0), not stored: NaN; (1, 1) stored: inf
    assert np.isnan(p[0]) and p[1] == np.inf
    # the same positions as CSR: row 0 stores column 0 twice
    b = csr(3, 2, [0, 2, 3, 4], [0, 0, 1, 0], [1.0, 5.0, 2.0, 7.0])
    assert R.partial(b, np.array([1.0, 1.0, 1.0]), True).tolist() == [5.0 + 7.0, 2.0]
    q = R.partial(b, np.array([-np.inf, 1.0, 1.0]), True)  # x[0] meets (0, 1), not stored
    assert q[0] == -np.inf and np.isnan(q[1])


def test_dense_partials_and_combination_order():
    A = np.array([[1e16, 1.0, -1e16], [-0.0, -0.0, -0.0]])
    x = np.ones(3)
    p = R.partial(dense(A), x, False)
    assert p[0] == 0.0 and p[1] == 0.0 and not np.signbit(p[1])   # ((0 + 1e16) + 1) - 1e16 = 0 (the 1 is absorbed)
    assert R.partial(dense(A, True), x, False).tolist() == p.tolist()
    assert R.partial(dense(A.T), x, True).tolist() == p.tolist()           # x A^T sums A's rows in the same order
    # partials combined left to right in k order
    S = R.combine([np.array([1e16]), np.array([1.0]), np.array([-1e16])])
    assert S[0] == 0.0
    S = R.combine([np.array([1.0]), np.array([1e16]), np.array([-1e16])])
    assert S[0] == 0.0
    S = R.combine([np.array([1e16]), np.array([-1e16]), np.array([1.0])])
    assert S[0] == 1.0

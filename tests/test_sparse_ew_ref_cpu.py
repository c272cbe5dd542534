"""CPU checks of tests/sparse_ew_ref.py: the golden TestSparse sums and Hadamard products, and hand-worked blocks for repeats,
-0.0 and non-finite values in both sparse (+) sparse branches and in dense (+) sparse."""
import json
import os

import numpy as np

from oracle import matrel_oracle as O
from tests import sparse_ew_ref as R

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "test_sparse.json")
NAN, INF = float("nan"), float("inf")


def csc(m, n, ptr, idx, val):
    return O.SparseMatrix(m, n, np.asarray(ptr, np.int32), np.asarray(idx, np.int32), np.asarray(val, np.float64), False)


def csr(m, n, ptr, idx, val):
    return O.SparseMatrix(m, n, np.asarray(ptr, np.int32), np.asarray(idx, np.int32), np.asarray(val, np.float64), True)


def same(a, b):
    return np.array_equal(R.bits(a), R.bits(b))


def test_golden_sum_and_hadamard():
    g = json.load(open(GOLDEN))
    s1, s2 = (csc(d["numRows"], d["numCols"], d["colPtrs"], d["rowIndices"], d["values"]) for d in (g["spmat1"], g["spmat2"]))
    fmt, v, _, _ = R.sparse_sparse("add", s1, s2)
    assert fmt == R.DENSE                     # 9 entries kept: 9 > 2 * 9 + 4 fails
    assert np.array_equal(v, np.asarray(g["expected"]["S1_plus_S2"]))
    fmt, v, ptr, idx = R.sparse_sparse("mul", s1, s2)
    assert fmt == R.CSC                       # one entry: 9 > 2 + 4
    want = np.asarray(g["expected"]["S1_hadamard_S2"])
    got = np.zeros((3, 3))
    for c in range(3):
        got[idx[ptr[c]:ptr[c + 1]], c] = v[ptr[c]:ptr[c + 1]]
    assert np.array_equal(got, want)
    # the same blocks as CSR (the transposes of their transposes' CSC arrays) take the toArray branch: the same values
    t1 = csr(3, 3, *R.to_sparse(R.to_array(s1).T))
    assert np.array_equal(R.to_array(t1), R.to_array(s1))
    fmt, v, _, _ = R.sparse_sparse("add", t1, s2)
    assert fmt == R.DENSE and np.array_equal(v, np.asarray(g["expected"]["S1_plus_S2"]))


def test_native_add_is_one_running_sum():
    # A(0,0) = 1, B(0,0) stored twice (1e16, -1e16): coltmp = ((0 + 1) + 1e16) - 1e16 = 0 (1 + 1e16 rounds to 1e16), dropped;
    # op(a, b) of the two sums would give 1
    a = csc(4, 4, [0, 1, 1, 1, 1], [0], [1.0])
    b = csc(4, 4, [0, 2, 2, 2, 2], [0, 0], [1e16, -1e16])
    fmt, v, ptr, idx = R.sparse_sparse("add", a, b)
    assert fmt == R.CSC and v.size == 0 and ptr.tolist() == [0, 0, 0, 0, 0]
    # multiply sums each operand on its own: (0 + 1) * ((0 + 1e16) - 1e16) = 0
    fmt, v, _, _ = R.sparse_sparse("mul", a, b)
    assert fmt == R.CSC and v.size == 0


def test_csc_repeats_sum_and_negative_zero():
    # repeats of a CSC operand are summed in storage order: 0.1 + 0.2 (rounded), not the last one
    a = csc(4, 4, [0, 2, 2, 2, 2], [1, 1], [0.1, 0.2])
    b = csc(4, 4, [0, 1, 1, 1, 1], [1], [2.0])
    fmt, v, ptr, idx = R.sparse_sparse("mul", a, b)
    assert fmt == R.CSC and idx.tolist() == [1] and v[0] == (0.0 + 0.1 + 0.2) * 2.0
    # a stored -0.0 becomes +0.0: (0.0 + -0.0) * -3 = -0.0, dropped; in a dense outcome it is +0.0
    a = csc(2, 2, [0, 1, 2], [0, 0], [-0.0, 5.0])
    b = csc(2, 2, [0, 1, 2], [0, 0], [-3.0, 7.0])
    fmt, v, _, _ = R.sparse_sparse("mul", a, b)
    assert fmt == R.DENSE                     # 4 > 2 * 1 + 3 fails
    assert same(v, np.array([[0.0, 35.0], [0.0, 0.0]]))


def test_csr_branch_last_wins_and_keeps_sign():
    # CSR row 0 stores column 1 twice: toArray keeps the last (3.0)
    a = csr(4, 4, [0, 2, 2, 2, 2], [1, 1], [2.0, 3.0])
    b = csc(4, 4, [0, 0, 1, 1, 1], [0], [5.0])
    fmt, v, ptr, idx = R.sparse_sparse("mul", a, b)
    assert fmt == R.CSC and idx.tolist() == [0] and v.tolist() == [15.0]
    # a CSC operand in this branch also keeps its last entry, not the sum
    a2 = csc(4, 4, [0, 0, 2, 2, 2], [0, 0], [2.0, 3.0])
    fmt, v, _, _ = R.sparse_sparse("add", a2, csr(4, 4, [0, 0, 0, 0, 0], [], []))
    assert fmt == R.CSC and v.tolist() == [3.0]
    # -0.0 kept where op makes it, in a dense outcome: -2 * (absent 0) = -0.0
    a = csr(2, 2, [0, 2, 4], [0, 1, 0, 1], [-2.0, 1.0, 1.0, 1.0])
    b = csr(2, 2, [0, 1, 3], [1, 0, 1], [4.0, 1.0, 1.0])
    fmt, v, _, _ = R.sparse_sparse("mul", a, b)
    assert fmt == R.DENSE and same(v, np.array([[-0.0, 4.0], [1.0, 1.0]]))


def test_non_finite_values():
    # case 2: Inf times an absent entry is NaN (kept); case 1 likewise (the other column holds 0.0)
    for a in (csr(4, 4, [0, 1, 1, 1, 1], [0], [INF]), csc(4, 4, [0, 1, 1, 1, 1], [0], [INF])):
        b = csc(4, 4, [0, 0, 1, 1, 1], [3], [1.0])
        fmt, v, ptr, idx = R.sparse_sparse("mul", a, b)
        assert fmt == R.CSC and ptr.tolist() == [0, 1, 1, 1, 1] and idx.tolist() == [0] and np.isnan(v[0])
    # divide: 0/0 everywhere nothing is stored, so the outcome is dense NaN with a/b at the union
    a = csc(2, 2, [0, 1, 1], [0], [1.0])
    b = csc(2, 2, [0, 1, 1], [0], [-0.5])
    fmt, v, _, _ = R.sparse_sparse("div", a, b)
    assert fmt == R.DENSE and v[0, 0] == -2.0 and np.isnan(v[1, 0]) and np.isnan(v[0, 1]) and np.isnan(v[1, 1])
    # NaN in a sum stays NaN; Inf - Inf is NaN
    a = csc(2, 2, [0, 1, 1], [0], [INF])
    b = csc(2, 2, [0, 1, 1], [0], [-INF])
    fmt, v, ptr, idx = R.sparse_sparse("add", a, b)
    assert fmt == R.DENSE and np.isnan(v[0, 0]) and same(v[:, 1], [0.0, 0.0])


def test_dense_sparse():
    d = O.DenseMatrix(2, 2, np.array([INF, -0.0, 4.0, 6.0]), False)          # column-major [[inf, 4], [-0, 6]]
    s = csr(2, 2, [0, 2, 3], [1, 1, 0], [2.0, 3.0, 0.5])                    # (0,1): 2 then 3 -> 3; (1,0): 0.5
    fmt, v, _, _ = R.dense_sparse("mul", d, s, False)
    assert fmt == R.DENSE and np.isnan(v[0, 0]) and same(v[:, 1], [12.0, 0.0]) and same([v[1, 0]], [-0.0 * 0.5])
    fmt, v, _, _ = R.dense_sparse("add", d, s, False)
    assert same(v, np.array([[INF, 7.0], [0.5, 6.0]]))                      # -0.0 + 0.5; 4 + 3
    fmt, v, _, _ = R.dense_sparse("div", d, s, False)                        # d / s: inf / 0 = inf, 6 / 0 = inf
    assert same(v, np.array([[INF, 4.0 / 3.0], [-0.0, INF]]))
    fmt, v, _, _ = R.dense_sparse("div", d, s, True)                         # s / d: 0 / inf = 0, 0.5 / -0 = -inf
    assert same(v, np.array([[0.0, 0.75], [-INF, 0.0]]))
    t = O.DenseMatrix(2, 2, np.array([INF, 4.0, -0.0, 6.0]), True)          # the same matrix, row-major
    assert same(R.dense_sparse("mul", t, s, False)[1], R.dense_sparse("mul", d, s, False)[1])

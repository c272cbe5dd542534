"""CPU checks of the sparse-product reference (tests/spmm_ref.py) on small hand-built blocks."""
import re
from fractions import Fraction

import numpy as np

from oracle import matrel_oracle as O
from tests.exact_ref import exact_dot
from tests.spmm_ref import (_CSRC, exact_sparse_entries, nonfinite_class, reference_product, segment_params,
                            sparse_sum_bound, within)


def csr(rows, cols, entries):
    """CSR block from per-row lists of (column, value), kept in the given order (duplicates and stored zeros allowed)."""
    ptr = np.cumsum([0] + [len(r) for r in entries])
    idx = [c for r in entries for c, _ in r]
    val = [v for r in entries for _, v in r]
    return O.SparseMatrix(rows, cols, ptr, np.array(idx, dtype=np.int32), np.array(val, dtype=np.float64), True)


def dense(a):
    a = np.asarray(a, dtype=np.float64)
    return O.DenseMatrix(a.shape[0], a.shape[1], np.ascontiguousarray(a.T).reshape(-1), False)


def small_product(rng):
    """2 x 2 block rows of blk 3 (ragged k: 5 columns): CSR, CSC and dense left blocks, one absent block."""
    blk, n, k, m = 3, 5, 5, 4
    Af = rng.uniform(-1, 1, (n, k)) * (rng.random((n, k)) < 0.5)
    A = {(0, 0): dense(Af[0:3, 0:3]).toSparse(),                                 # CSC
         (0, 1): dense(Af[0:3, 3:5]),
         (1, 0): dense(Af[3:5, 0:3].T).toSparse().transpose()}                    # CSR
    Af[3:5, 3:5] = 0.0                                                           # block (1, 1) absent
    Bf = rng.uniform(-1, 1, (k, m))
    B = {(0, 0): dense(Bf[0:3, 0:3]), (0, 1): dense(Bf[0:3, 3:4]), (1, 0): dense(Bf[3:5, 0:3]), (1, 1): dense(Bf[3:5, 3:4])}
    return A, B, Af, Bf, n, k, m, blk


def test_exact_entries_equal_the_dense_images_for_finite_data():
    rng = np.random.default_rng(1)
    A, B, Af, Bf, n, k, m, blk = small_product(rng)
    assert A[(1, 0)].isTransposed and not A[(0, 0)].isTransposed
    pos = [(i, j) for i in range(n) for j in range(m)]
    got = exact_sparse_entries(A, B, n, k, m, blk, pos)
    assert got == [exact_dot(Af[i, :], Bf[:, j]) for i, j in pos]
    C = reference_product(A, B, n, k, m, blk)
    assert np.all(np.abs(C - Af @ Bf) <= sparse_sum_bound(A, B, n, k, m, blk))


def test_duplicates_and_stored_zeros_are_terms():
    A = {(0, 0): csr(2, 3, [[(2, 0.5), (0, 1.0), (2, 0.25)], [(1, 0.0)]])}
    B = {(0, 0): dense([[1.0], [np.inf], [3.0]])}
    assert exact_sparse_entries(A, B, 2, 3, 1, 4, [(0, 0)]) == [Fraction(1) + Fraction(9, 4)]
    assert nonfinite_class(A, B, 2, 3, 1, 4, [(0, 0), (1, 0)]) == ["finite", "nan"]     # Inf x a stored 0.0
    S = sparse_sum_bound(A, B, 2, 3, 1, 4)
    assert S[0, 0] == 1.01 * 5 * 2.0 ** -53 * 3.25 + 7 * 2.0 ** -1074                  # three terms
    C = reference_product(A, B, 2, 3, 1, 4)
    assert C[0, 0] == 3.25 and np.isnan(C[1, 0])


def test_nan_in_an_unreferenced_row_of_b_stays_out():
    A = {(0, 0): csr(2, 4, [[(0, 2.0), (3, -1.0)], []])}
    B = {(0, 0): dense([[1.0, 1.0], [np.nan, np.inf], [-np.inf, np.nan], [4.0, -np.inf]])}
    pos = [(0, 0), (0, 1), (1, 0), (1, 1)]
    assert nonfinite_class(A, B, 2, 4, 2, 4, pos) == ["finite", "+inf", "finite", "finite"]
    C = reference_product(A, B, 2, 4, 2, 4)
    assert C[0, 0] == -2.0 and C[0, 1] == np.inf and C[1, 0] == 0.0 and C[1, 1] == 0.0


def test_bound_rejects_a_result_just_outside_and_accepts_one_just_inside():
    rng = np.random.default_rng(2)
    A, B, Af, Bf, n, k, m, blk = small_product(rng)
    S = sparse_sum_bound(A, B, n, k, m, blk)
    pos = [(i, j) for i in range(n) for j in range(m)]
    for (i, j), x in zip(pos, exact_sparse_entries(A, B, n, k, m, blk, pos)):
        for sign in (1, -1):
            edge = float(x + sign * Fraction(float(S[i, j])))        # the doubles on either side of exact +- bound
            near = [np.nextafter(edge, -np.inf), edge, np.nextafter(edge, np.inf)]
            ok = [within(v, x, S[i, j]) for v in near]
            assert ok in ([True, True, False], [True, False, False]) if sign > 0 else ok in ([False, True, True], [False, False, True])
    # a dropped, a doubled and a misplaced entry each move the sum far outside the bound
    rows = [[(0, 0.75), (2, -0.5), (3, 0.125)]]
    B1 = {(0, 0): dense(rng.uniform(0.5, 1, (4, 3)))}
    S1 = sparse_sum_bound({(0, 0): csr(1, 4, rows)}, B1, 1, 4, 3, 4)
    exact = np.array([float(x) for x in exact_sparse_entries({(0, 0): csr(1, 4, rows)}, B1, 1, 4, 3, 4, [(0, j) for j in range(3)])])
    for wrong in ([rows[0][:2]], [rows[0] + rows[0][2:]], [[(0, 0.75), (1, -0.5), (3, 0.125)]]):
        got = reference_product({(0, 0): csr(1, 4, wrong)}, B1, 1, 4, 3, 4)[0]
        assert np.all(np.abs(got - exact) > S1[0])


def test_segment_constants_match_the_kernel_static_asserts():
    p = segment_params()
    src = open(f"{_CSRC}/spmm.cu").read()
    assert "static_assert(TN == 64 && RPW == 16" in src and "constexpr int RPW = TM / NCW;" in src
    assert p["TN"] == 64 and p["TM"] // p["NCW"] == 16 and p["TM"] % p["NCW"] == 0
    assert p["KC"] > 0 and p["KC"] % 32 == 0
    # the shared-memory budget the third static_assert checks, from the same constants
    stage = p["KC"] * p["TN"] * 8 + p["E_CAP"] * 16 + (p["TM"] + 4) * 4
    nstage = int(re.search(r"constexpr int NSTAGE = (\d+);", src).group(1))
    assert 128 + nstage * ((stage + 127) // 128 * 128) + 64 <= 227 * 1024
    assert (p["TM"] + 1) * p["TN"] * 8 <= nstage * ((stage + 127) // 128 * 128)

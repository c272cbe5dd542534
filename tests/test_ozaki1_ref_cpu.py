"""CPU checks of the Ozaki-I model and bound (tests/ozaki1_ref.py), no GPU needed.

- The model is exact where the arithmetic must be exact, and within ozaki1_bound on adversarial data (digit-saturating values,
  alternating signs, K at the s32 accumulator limit, lines of tiny and huge magnitude).
- Planted errors -- a dropped diagonal, a wrong digit pair, the exponent without its + 1, truncated digits, a row-major block
  read with the column-major stride -- change the model's bits, and most of them leave the bound.
- The epilogue the library had before scaled each term by (2^e_i 2^(4-8d)) 2^f_j: the row factor is +inf for a row maximum of
  2^1023 or more, and underflows for rows of tiny magnitude.  Replayed here, that epilogue gives inf / NaN or loses diagonals on
  such rows although the product is an ordinary number, and those results are outside the bound."""
from fractions import Fraction

import numpy as np
import pytest

from oracle import matrel_oracle as O
from tests.exact_ref import exact_entries, round_to_double
from tests.ozaki1_ref import (clamp_slices, diagonals, digits, epilogue, line_exponents, ozaki1_bound, ozaki1_model,
                              seen_operands)

TINY = 2.0 ** -1074


def all_pos(C):
    return [(i, j) for i in range(C.shape[0]) for j in range(C.shape[1])]


def worst_ratio(C, A, B, S):
    """max |C - exact| / bound over every entry (inf when a non-finite C meets a finite exact product)."""
    bound = ozaki1_bound(A, B, S, np.zeros(C.shape))
    worst = 0.0
    for (i, j), x in zip(all_pos(C), exact_entries(A, B, all_pos(C))):
        want = round_to_double(x)
        lim = Fraction(float(bound[i, j])) + Fraction(2.0 ** -52 * abs(want))
        if not np.isfinite(C[i, j]):
            return np.inf
        worst = max(worst, float(abs(Fraction(float(C[i, j])) - x) / lim))
    return worst


def legacy_model(A, B, S):
    """The epilogue the library had: term = (acc (2^e_i 2^(4-8d))) 2^f_j in fp64, with 2^e = scalbn(1, e)."""
    e, f = line_exponents(A, 1), line_exponents(B, 0)
    acc = diagonals(digits(A, e, S), digits(B.T, f, S), S)
    C = None
    with np.errstate(over="ignore", under="ignore", invalid="ignore"):
        rs0, cs = np.ldexp(1.0, e), np.ldexp(1.0, f)
        for d in range(S + 1, 1, -1):
            t = (acc[d] * (rs0 * 2.0 ** (4 - 8 * d))[:, None]) * cs[None, :]
            C = t if C is None else C + t
    return C


# ------------------------------------------------------------------------------------------------ the model's own steps
def test_ldexp_rounds_once_like_the_device():
    """Step 4 relies on np.ldexp rounding acc 2^n correctly, ties to even, into the sub-normal range and to zero."""
    rng = np.random.default_rng(1)
    accs = [1, -1, 3, 5, -7, (1 << 31) - 1, -(1 << 31) + 1] + rng.integers(-(1 << 31) + 1, 1 << 31, 200).tolist()
    for a in accs:
        for n in [-1074, -1075, -1076, -1100, -1104, -1105, -1106, -2044, -2045, -2206, -1022, -1040, 900, 992, 993, 2036] + \
                 rng.integers(-1110, -1040, 3).tolist():
            with np.errstate(over="ignore", under="ignore"):
                got = np.ldexp(float(a), n)
            assert got == round_to_double(Fraction(a) * Fraction(2) ** n), (a, n)
            if got == 0.0:
                assert np.signbit(got) == (a < 0)


@pytest.mark.parametrize("S", [2, 3, 4, 5, 6, 7])
def test_digits_reconstruct_the_rounded_operand(S):
    rng = np.random.default_rng(S)
    L = rng.uniform(-1, 1, (6, 40)) * np.exp2(rng.integers(-1070, 1000, 6))[:, None]
    L[0, :3] = [np.nextafter(1.0, 0.0), -np.nextafter(1.0, 0.0), 0.5]
    L[1] = TINY * rng.integers(-9, 9, 40)
    e = line_exponents(L, 1)
    D = digits(L, e, S)
    assert D.min() >= -128 and D.max() <= 127 and np.abs(D[0]).max() <= 64      # the top digit holds |X| <= 2^(8S-2)
    for i in range(L.shape[0]):
        for k in range(L.shape[1]):
            X = sum(int(D[s, i, k]) << (8 * (S - 1 - s)) for s in range(S))
            want = round(Fraction(float(L[i, k])) * Fraction(2) ** (8 * S - 2 - int(e[i])))   # Python round(): ties to even
            assert X == want


def test_slice_clamps():
    assert [clamp_slices(s) for s in (0, 1, 2, 7, 8, 9)] == [7, 2, 2, 7, 7, 7]


# ------------------------------------------------------------------------------------------------ exactness
@pytest.mark.parametrize("S", [2, 4, 7])
def test_one_nonzero_digit_is_exact(S):
    """a = c 2^(e-6) with |c| <= 63 and a line maximum of |c| >= 32: X = c 256^(S-1), one digit, and only diagonal 2 is non-zero."""
    rng = np.random.default_rng(10 + S)
    n, K, m = 9, 300, 7
    A = rng.integers(-63, 64, (n, K)).astype(np.float64)
    B = rng.integers(-63, 64, (K, m)).astype(np.float64)
    A[:, 0], B[0, :] = 63.0, -40.0
    A *= np.exp2(rng.integers(-1000, 900, n))[:, None]
    B *= np.exp2(rng.integers(-60, 60, m))[None, :]
    C = ozaki1_model(A, B, S)
    assert np.array_equal(C, np.array([round_to_double(x) for x in exact_entries(A, B, all_pos(C))]).reshape(C.shape))


def test_short_integers_are_exact():
    """|a|, |b| < 2^20: three digits each, no diagonal beyond S + 1 = 8 is dropped, every sum is an exact fp64 integer."""
    rng = np.random.default_rng(3)
    A = rng.integers(-(1 << 20) + 1, 1 << 20, (12, 500)).astype(np.float64)
    B = rng.integers(-(1 << 20) + 1, 1 << 20, (500, 11)).astype(np.float64)
    C = ozaki1_model(A, B, 7)
    assert np.array_equal(C, (A.astype(object) @ B.astype(object)).astype(np.float64))


# ------------------------------------------------------------------------------------------------ adversarial data
def saturating(rng, n, K, sign, S):
    """Lines of one value whose S - 1 low digits are all -128 (|digit product| = 2^14, the most an accumulator term can be) and whose
    top digit is 64 (-63 for the negated value): X = 64 256^(S-1) - 128 (256^(S-1) - 1) / 255, just below 2^(8S-2), even, so exact in fp64 for S = 7 too."""
    X = 64 * 256 ** (S - 1) - 128 * (256 ** (S - 1) - 1) // 255
    q = rng.integers(-40, 40, n)
    return sign * np.ldexp(float(X), q + 2 - 8 * S)[:, None] * np.ones((n, K))


@pytest.mark.parametrize("S", [2, 5, 7])
def test_accumulator_limit_with_saturating_digits(S):
    """The largest K with K S < 2^17 (the rule of try_ozaki): every accumulator stays below 2^31 and the result within the bound."""
    K = ((1 << 17) - 1) // S
    rng = np.random.default_rng(S)
    alt = np.where(np.arange(K) % 2 == 0, 1.0, -1.0)
    A = np.vstack([saturating(rng, 2, K, 1.0, S), saturating(rng, 1, K, alt[None, :], S)])
    B = np.vstack([saturating(rng, 2, K, -1.0, S), saturating(rng, 1, K, 1.0, S)]).T
    e, f = line_exponents(A, 1), line_exponents(B, 0)
    DA, DB = digits(A, e, S), digits(B.T, f, S)
    assert np.abs(DA[1:]).min() >= 127 and np.abs(DB[1:]).min() >= 127 and np.abs(DA[0]).min() >= 63
    acc = diagonals(DA, DB, S)
    assert 2.0 ** 29 < max(np.abs(a).max() for a in acc.values()) < 2.0 ** 31
    assert K * S < (1 << 17) <= (K + 1) * S
    assert worst_ratio(epilogue(acc, e, f, S), A, B, S) <= 1.0


@pytest.mark.parametrize("S", [2, 3, 7])
def test_wide_ranges_and_cancellation_within_the_bound(S):
    rng = np.random.default_rng(20 + S)
    n, K, m = 8, 90, 6
    A = rng.uniform(-1, 1, (n, K)) * np.exp2(rng.integers(-300, 300, (n, K)))   # 2^+-300 inside each line
    B = rng.uniform(-1, 1, (K, m)) * np.exp2(rng.integers(-300, 300, (K, m)))
    A[0] = np.where(np.arange(K) % 2, 1.0, -1.0) * np.nextafter(1.0, 0.0)        # alternating signs: the product cancels
    B[:, 0] = 1.0 / 3.0
    A[1, :] = 0.0
    A[2] = rng.uniform(-1, 1, K) * 2.0 ** 700                                    # products up to 2^1000
    A[3] = A[3] * 2.0 ** -1000                                                   # sub-normal and tiny rows
    A[4] = TINY * rng.integers(-1000, 1000, K)
    B[:, 1] = rng.uniform(-1, 1, K) * 2.0 ** -20
    assert worst_ratio(ozaki1_model(A, B, S), A, B, S) <= 1.0


# ------------------------------------------------------------------------------------------------ planted errors
def plant(A, B, S, what):
    e, f = line_exponents(A, 1), line_exponents(B, 0)
    if what == "no_plus_one":                          # e = ilogb(max): X reaches 2^(8S-1), beyond S balanced digits
        e, f = e - 1, f - 1
        with np.errstate(under="ignore"):
            XA = np.rint(np.ldexp(A, (8 * S - 2 - e)[:, None])).astype(np.int64)
            XB = np.rint(np.ldexp(B.T, (8 * S - 2 - f)[:, None])).astype(np.int64)

        def dig(X):                                    # the carry out of the top digit is lost, as in slice_kernel
            out = np.empty((S,) + X.shape, dtype=np.int64)
            for s in range(S, 0, -1):
                dgt = ((X + 128) & 255) - 128
                X = (X - dgt) >> 8
                out[s - 1] = dgt
            return out
        return epilogue(diagonals(dig(XA), dig(XB), S), e, f, S)
    if what == "truncated_digit":
        def dig(L, ex):
            X = np.trunc(np.ldexp(L, (8 * S - 2 - ex)[:, None])).astype(np.int64)
            out = np.empty((S,) + L.shape, dtype=np.int64)
            for s in range(S, 0, -1):
                dgt = ((X + 128) & 255) - 128
                X = (X - dgt) >> 8
                out[s - 1] = dgt
            return out
        return epilogue(diagonals(dig(A, e), dig(B.T, f), S), e, f, S)
    DA, DB = digits(A, e, S), digits(B.T, f, S)
    acc = diagonals(DA, DB, S)
    if what == "dropped_diagonal":                     # the smallest diagonal S + 1 left out
        acc[S + 1] = np.zeros_like(acc[S + 1])
    elif what == "wrong_pair":                         # diagonal 3 pairs (1, 2) with (1, 1) instead of (2, 1)
        fa, fb = DA.astype(float), DB.astype(float)
        acc[3] = fa[0] @ fb[1].T + fa[0] @ fb[0].T
    return epilogue(acc, e, f, S)


@pytest.mark.parametrize("S", [3, 7])
@pytest.mark.parametrize("what,leaves_bound", [("dropped_diagonal", True), ("wrong_pair", True), ("no_plus_one", True),
                                                ("truncated_digit", False)])
def test_planted_errors_are_caught(S, what, leaves_bound):
    rng = np.random.default_rng(S)
    n, K, m = 6, 64, 5
    A = rng.uniform(0.5, 1.0, (n, K)) * np.exp2(rng.integers(-20, 20, n))[:, None] * np.exp2(rng.integers(-12, 0, (n, K)))
    B = rng.uniform(0.5, 1.0, (K, m)) * np.exp2(rng.integers(-12, 0, (K, m)))
    A[:, 0] = np.nextafter(np.exp2(np.floor(np.log2(A.max(axis=1)))) * 2, 0.0)   # line maxima just below a power of two
    B[0, :] = -np.nextafter(1.0, 0.0)
    good, bad = ozaki1_model(A, B, S), plant(A, B, S, what)
    assert worst_ratio(good, A, B, S) <= 1.0
    assert not np.array_equal(good, bad)
    if leaves_bound:
        assert worst_ratio(bad, A, B, S) > 1.0


def test_row_major_block_read_with_the_column_major_stride_is_caught():
    rng = np.random.default_rng(5)
    n, blk = 48, 16
    Af, Bf = rng.uniform(-1, 1, (n, n)), rng.uniform(-1, 1, (n, n))
    A = {(i, j): O.DenseMatrix(blk, blk, np.ascontiguousarray(Af[i * blk:(i + 1) * blk, j * blk:(j + 1) * blk]).reshape(-1), True)
         for i in range(3) for j in range(3)}
    B = {(i, j): O.DenseMatrix(blk, blk, np.ascontiguousarray(Bf[i * blk:(i + 1) * blk, j * blk:(j + 1) * blk].T).reshape(-1))
         for i in range(3) for j in range(3)}
    sa, sb = seen_operands(A, B, n, n, n, blk)
    assert np.array_equal(sa, Af) and np.array_equal(sb, Bf)
    wrong = dict(A)
    wrong[(1, 2)] = O.DenseMatrix(blk, blk, A[(1, 2)].values, False)               # the same storage, read column-major
    wa, _ = seen_operands(wrong, B, n, n, n, blk)
    bad = ozaki1_model(wa, Bf, 7)
    assert not np.array_equal(bad, ozaki1_model(Af, Bf, 7))
    assert worst_ratio(bad, Af, Bf, 7) > 1.0


def test_blocks_that_meet_nothing_set_no_exponent():
    """A block of A whose k has no block of B is not an operand of the kernel: a huge value there leaves its row's exponent."""
    rng = np.random.default_rng(6)
    n, blk = 40, 16
    Af, Bf = rng.uniform(-1, 1, (n, n)), rng.uniform(-1, 1, (n, n))
    Af[3, 2 * blk + 1] = 2.0 ** 900
    A = {(i, j): O.DenseMatrix(*Af[i * blk:(i + 1) * blk, j * blk:(j + 1) * blk].shape,
                               np.ascontiguousarray(Af[i * blk:(i + 1) * blk, j * blk:(j + 1) * blk].T).reshape(-1))
         for i in range(3) for j in range(3)}
    B = {(i, j): O.DenseMatrix(*Bf[i * blk:(i + 1) * blk, j * blk:(j + 1) * blk].shape,
                               np.ascontiguousarray(Bf[i * blk:(i + 1) * blk, j * blk:(j + 1) * blk].T).reshape(-1))
         for i in range(2) for j in range(3)}                                      # block row k = 2 of B is absent
    sa, sb = seen_operands(A, B, n, n, n, blk)
    assert sa[3, 2 * blk + 1] == 0.0 and line_exponents(sa, 1)[3] == line_exponents(Af[:, :2 * blk], 1)[3]
    assert np.array_equal(sb[2 * blk:], np.zeros((n - 2 * blk, n)))


# ------------------------------------------------------------------------------------------------ the two-factor epilogue
def test_two_factor_scaling_overflows_on_rows_at_the_top_of_the_range():
    """A row holding 1.5 2^1023 times a column of 2^-1000 values: e = 1024 makes 2^e = +inf, so every term is +-inf or NaN."""
    rng = np.random.default_rng(7)
    K = 40
    A = rng.uniform(-1, 1, (3, K))
    A[0, 5] = 1.5 * 2.0 ** 1023
    A[1] = rng.uniform(1, 1.9, K) * 2.0 ** 1023
    B = rng.uniform(-1, 1, (K, 3)) * 2.0 ** -1000
    B[:, 2] = 2.0 ** -1000
    for S in (2, 7):
        old, new = legacy_model(A, B, S), ozaki1_model(A, B, S)
        assert not np.isfinite(old[:2]).any() and np.isnan(old[:2]).any()
        assert np.isfinite(new).all() and worst_ratio(new, A, B, S) <= 1.0
        assert worst_ratio(old, A, B, S) == np.inf


@pytest.mark.parametrize("lo,hi", [(-1016, -1015), (-1040, -1016), (-1060, -1040)])
def test_two_factor_scaling_loses_diagonals_on_tiny_rows(lo, hi):
    """Rows of tiny normal values times columns near 2^1000: 2^e_i 2^(4-8d) underflows for the small diagonals."""
    rng = np.random.default_rng(-lo)
    K = 64
    A = rng.uniform(1, 2, (4, K)) * np.exp2(rng.integers(lo, hi, (4, K)).astype(float))
    B = rng.uniform(-1, 1, (K, 3)) * 2.0 ** 1000
    S = 7
    old, new = legacy_model(A, B, S), ozaki1_model(A, B, S)
    assert worst_ratio(new, A, B, S) <= 1.0
    assert worst_ratio(old, A, B, S) > 1.0
    assert worst_ratio(legacy_model(B.T, A.T, S), B.T, A.T, S) <= 1.0      # the mirror case: the column factor comes last


def test_two_factor_scaling_loses_everything_but_one_diagonal_on_subnormal_rows():
    rng = np.random.default_rng(9)
    K = 64
    A = TINY * rng.integers(1 << 20, 1 << 30, (3, K)).astype(float)
    B = rng.uniform(-1, 1, (K, 2)) * 2.0 ** 1000
    old, new = legacy_model(A, B, 7), ozaki1_model(A, B, 7)
    assert worst_ratio(new, A, B, 7) <= 1.0
    assert worst_ratio(old, A, B, 7) > 1e6


# ------------------------------------------------------------------------------------------------ results near the top of the range
DBL_MAX = np.finfo(np.float64).max
NO_SCALING = 4096                                  # above every e_i + f_j: the epilogue without its scaled sums


def test_a_product_just_below_the_largest_double_is_finite():
    """a b = 1.7887e308, 0.5 % below the largest double: the top-digit term t_2 alone overshoots the fp64 range, so without the
    scaled sums the product would be +inf."""
    A, B = np.array([[6.703903964971299e153]]), np.array([[2.6681537780585762e154]])
    for S in range(2, 8):
        assert worst_ratio(ozaki1_model(A, B, S), A, B, S) <= 1.0
        e, f = line_exponents(A, 1), line_exponents(B, 0)
        acc = diagonals(digits(A, e, S), digits(B.T, f, S), S)
        assert np.isinf(epilogue(acc, e, f, S, scaled_above=NO_SCALING)).all()


@pytest.mark.parametrize("S", [2, 3, 5, 7])
def test_products_at_0995_of_the_largest_double_are_finite_and_within_the_bound(S):
    """a over [1, 2) 2^511, b = 0.995 DBL_MAX / a: every product is finite and within the bound, where the unscaled sums give +inf
    for a good share of them."""
    rng = np.random.default_rng(S)
    a = np.ldexp(rng.uniform(1, 2, 400), 511)
    b = 0.995 * DBL_MAX / a
    A, B = a[:, None], b[None, :]
    e, f = line_exponents(A, 1), line_exponents(B, 0)
    acc = diagonals(digits(A, e, S), digits(B.T, f, S), S)
    C, old = np.diag(epilogue(acc, e, f, S)), np.diag(epilogue(acc, e, f, S, scaled_above=NO_SCALING))
    bound = np.diag(ozaki1_bound(A, B, S, np.zeros((400, 400))))
    assert np.isfinite(C).all() and np.isinf(old).sum() > 20
    for i in range(400):
        x = Fraction(float(a[i])) * Fraction(float(b[i]))
        assert abs(Fraction(float(C[i])) - x) <= Fraction(float(bound[i])) + Fraction(2.0 ** -52) * x


@pytest.mark.parametrize("S", [2, 4, 7])
def test_scaled_sums_change_no_bit_below_the_overflow(S):
    """For e_i + f_j just below and above the threshold, the scaled sums give the unscaled result bit for bit (no term
    is near the sub-normals, so the scaling by 2^-(e_i + f_j) is exact), sub-normal and zero products included."""
    rng = np.random.default_rng(30 + S)
    K = 50
    A = rng.uniform(-1, 1, (6, K)) * np.exp2(np.array([-1000, 0, 480, 500, 501, 510], dtype=float))[:, None]
    B = rng.uniform(-1, 1, (K, 5)) * np.exp2(np.array([-60, 10, 499, 500, 501], dtype=float))[None, :]
    B[:, 0] = 0.0
    e, f = line_exponents(A, 1), line_exponents(B, 0)
    assert ((e[:, None] + f[None, :]) == 1000).any() and ((e[:, None] + f[None, :]) == 1001).any()
    acc = diagonals(digits(A, e, S), digits(B.T, f, S), S)
    new, old = epilogue(acc, e, f, S), epilogue(acc, e, f, S, scaled_above=NO_SCALING)
    assert np.isfinite(old).all() and np.array_equal(new.view(np.int64), old.view(np.int64))

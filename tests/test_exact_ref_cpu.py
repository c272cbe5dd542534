"""CPU checks of tests/exact_ref.py: the exact dot product against brute-force Fraction sums, the correctly rounded conversion,
and numpy's fp64 product against the classical bound relative to the exact one."""
import math
from fractions import Fraction

import numpy as np
import pytest

from tests.exact_ref import (alpha_of, exact_dot, exact_entries, fp64_dot_bound, moduli_for, oz2_bound, round_to_double)
from tests.test_crt_math_cpu import alpha_of as alpha_rule

TINY = 2.0 ** -1074


def brute(a, b):
    return sum((Fraction(float(x)) * Fraction(float(y)) for x, y in zip(a, b)), Fraction(0))


def vectors(kind, rng, k):
    if kind == "random":
        return rng.uniform(-1, 1, k), rng.uniform(-1, 1, k)
    if kind == "subnormal":
        return rng.integers(-(1 << 40), 1 << 40, k) * TINY, rng.uniform(-2, 2, k)
    if kind == "mixed_subnormal":
        a = rng.uniform(-1, 1, k)
        a[::3] = rng.integers(1, 1 << 20, a[::3].size) * TINY
        return a, rng.uniform(-1, 1, k) * np.exp2(rng.integers(-1000, 1000, k))
    if kind == "huge":
        return rng.uniform(-1, 1, k) * 2.0 ** 1023, rng.uniform(-1, 1, k) * 2.0 ** 1023
    if kind == "wide":
        return (rng.uniform(-1, 1, k) * np.exp2(rng.integers(-1070, 1023, k)),
                rng.uniform(-1, 1, k) * np.exp2(rng.integers(-1070, 1023, k)))
    if kind == "cancelling":
        a = rng.uniform(1, 2, k)
        b = rng.uniform(1, 2, k)
        a[1::2], b[1::2] = -a[0::2][:a[1::2].size], b[0::2][:b[1::2].size]
        return a, b
    if kind == "zeros":
        a = rng.uniform(-1, 1, k)
        a[rng.random(k) < 0.5] = 0.0
        a[0] = -0.0
        return a, rng.uniform(-1, 1, k)
    raise AssertionError(kind)


@pytest.mark.parametrize("kind", ["random", "subnormal", "mixed_subnormal", "huge", "wide", "cancelling", "zeros"])
@pytest.mark.parametrize("k", [1, 2, 7, 64])
def test_exact_dot_equals_the_fraction_sum(kind, k):
    rng = np.random.default_rng(k * 131 + len(kind))
    for _ in range(5):
        a, b = vectors(kind, rng, k)
        assert exact_dot(a, b) == brute(a, b)


def test_exact_entries_index_rows_of_a_and_columns_of_b():
    rng = np.random.default_rng(3)
    A, B = rng.uniform(-1, 1, (5, 9)), rng.uniform(-1, 1, (9, 4))
    pairs = [(0, 0), (4, 3), (2, 1)]
    assert exact_entries(A, B, pairs) == [brute(A[i], B[:, j]) for i, j in pairs]
    assert exact_entries(np.zeros((2, 3)), B[:3], [(1, 2)]) == [Fraction(0)]
    with pytest.raises(AssertionError):
        exact_entries(np.array([[np.inf]]), np.array([[1.0]]), [(0, 0)])


def test_cancellation_keeps_the_last_bit():
    a = np.array([2.0 ** 60, 1.0, -2.0 ** 60])
    b = np.array([1.0, 2.0 ** -60, 1.0])
    assert exact_dot(a, b) == Fraction(1, 1 << 60)
    assert float(a @ b) == 0.0                       # fp64 loses it; the reference does not


def test_round_to_double():
    assert round_to_double(Fraction(1, 3)) == 1.0 / 3.0
    assert round_to_double(Fraction(2) ** 1024) == math.inf and round_to_double(-Fraction(2) ** 1024) == -math.inf
    top = Fraction(float(np.finfo(np.float64).max))
    half_ulp = Fraction(2) ** 970
    assert round_to_double(top + half_ulp / 2) == float(top)
    assert round_to_double(top + half_ulp) == math.inf          # the tie rounds to the even neighbour, which is 2^1024
    assert round_to_double(Fraction(3, 2) * Fraction(2) ** -1074) == 2 * TINY   # tie to even in the sub-normal range
    assert round_to_double(Fraction(1, 2) * Fraction(2) ** -1074) == 0.0
    assert round_to_double(Fraction(1) + Fraction(2) ** -53) == 1.0 and round_to_double(Fraction(1) + Fraction(2) ** -53 + Fraction(2) ** -80) > 1.0


@pytest.mark.parametrize("kind", ["random", "wide_rows", "cancelling"])
def test_numpy_product_meets_the_classical_bound(kind):
    rng = np.random.default_rng(11)
    n, k, m = 12, 300, 9
    A, B = rng.uniform(-1, 1, (n, k)), rng.uniform(-1, 1, (k, m))
    if kind == "wide_rows":
        A *= np.exp2(rng.integers(-300, 300, n))[:, None]
    if kind == "cancelling":
        A[:, 1::2], B[1::2, :] = -A[:, 0::2], B[0::2, :]
    got, bound = A @ B, fp64_dot_bound(A, B)
    pairs = [(i, j) for i in range(n) for j in range(m)]
    for (i, j), x in zip(pairs, exact_entries(A, B, pairs)):
        assert abs(Fraction(float(got[i, j])) - x) <= Fraction(float(bound[i, j])), (i, j)


def test_alpha_and_moduli_rules():
    for T in range(6, 17):
        for K in (1, 2, 3, 255, 256, 257, 1000, 4096, 4097, 65536, 131071):
            assert alpha_of(T, K) == alpha_rule(T, K)[0]
    assert all(moduli_for(K) == 14 for K in (256, 1000, 4096, 16384, 65536, 131071))
    assert moduli_for(1000, 16) == 16 and moduli_for(1000, 3) == 6 and moduli_for(1000, 99) == 16
    assert alpha_of(14, 16384) == 47 and alpha_of(16, 16384) == 55


def test_oz2_bound_covers_operands_rounded_to_alpha_bits():
    """Emulate the scheme in exact arithmetic (round every line to alpha bits below a power of two above its maximum, multiply
    exactly, round once): the error stays inside oz2_bound, and a further error of one part in 2^(alpha - 6) does not."""
    rng = np.random.default_rng(5)
    n, k, m, alpha = 6, 40, 5, 30
    A = rng.uniform(-1, 1, (n, k)) * np.exp2(rng.integers(-30, 30, n))[:, None]
    B = rng.uniform(-1, 1, (k, m)) * np.exp2(rng.integers(-30, 30, m))[None, :]
    ea = np.frexp(np.abs(A).max(axis=1))[1]
    eb = np.frexp(np.abs(B).max(axis=0))[1]
    Ar = np.rint(np.ldexp(A, (alpha - ea)[:, None])) * np.exp2(ea - alpha)[:, None]
    Br = np.rint(np.ldexp(B, (alpha - eb)[None, :])) * np.exp2(eb - alpha)[None, :]
    pairs = [(i, j) for i in range(n) for j in range(m)]
    exact = exact_entries(A, B, pairs)
    scheme = [round_to_double(x) for x in exact_entries(Ar, Br, pairs)]
    bound = oz2_bound(A, B, alpha, A @ B)
    absAB = np.abs(A) @ np.abs(B)
    worst = 0.0
    for (i, j), x, g in zip(pairs, exact, scheme):
        err = abs(Fraction(g) - x)
        assert err <= Fraction(float(bound[i, j])), (i, j)
        worst = max(worst, float(err) / float(bound[i, j]))
        assert float(absAB[i, j]) * 2.0 ** -(alpha - 6) > float(bound[i, j])      # a kernel 6 bits short would be caught
    assert worst > 0.01                                                        # the bound is not slack by orders of magnitude

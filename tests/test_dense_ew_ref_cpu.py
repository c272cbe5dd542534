"""CPU checks of tests/dense_ew_ref.py: the exact sums and the summation bound accept every summation order and reject planted
errors (a term dropped, a term counted twice, a row read with the other layout's stride); the rank-one reference rejects a fused
multiply-add; java_pow follows the specification of java.lang.Math.pow, C's pow does not, and the oracle's matrixPow agrees with
java_pow."""
import math
from fractions import Fraction

import numpy as np
import pytest

from oracle import matrel_oracle as O
from tests import dense_ew_ref as R

NAN, INF = math.nan, math.inf
TINY = 5e-324  # the smallest subnormal


def same(a, b):
    return np.array_equal(R.bits(a), R.bits(b))


def block(a, rowmajor):
    a = np.asarray(a, dtype=np.float64)
    return O.DenseMatrix(a.shape[0], a.shape[1], np.ascontiguousarray(a if rowmajor else a.T).reshape(-1), rowmajor)


def orders(rng, x):
    """Sums of x in several orders, each add rounded: left to right, right to left, numpy's pairwise sum, shuffled, and the
    dense kernels' shapes (8 and 32 strided partials folded, then atomics in a shuffled order)."""
    out = []
    for seq in (x, x[::-1], x[rng.permutation(x.size)]):
        s = 0.0
        for v in seq.tolist():
            s += v
        out.append(s)
    out.append(float(np.sum(x)))
    for lanes in (8, 32):
        parts = []
        for lane in range(lanes):
            s = 0.0
            for v in x[lane::lanes].tolist():
                s += v
            parts.append(s)
        s = 0.0
        for p in rng.permutation(parts).tolist():
            s += p
        out.append(s)
    return out


def test_int_sums_are_every_order():
    rng = np.random.default_rng(1)
    T = rng.integers(-2 ** 30, 2 ** 30, (20, 1025)).astype(np.float64)
    want = R.int_sums(T)
    for t in range(T.shape[0]):
        assert want[t] == math.fsum(T[t].tolist())
        assert all(s == want[t] for s in orders(rng, T[t]))
    assert same(R.int_sums(np.array([[-0.0, -0.0], [3.0, -3.0]])), [0.0, 0.0])  # sums start at +0.0
    with pytest.raises(AssertionError):
        R.int_sums(np.array([[0.5, 1.0]]))
    with pytest.raises(AssertionError):
        R.int_sums(np.array([[2.0 ** 52, 2.0 ** 52]]))


def test_bound_accepts_every_order():
    rng = np.random.default_rng(2)
    for n in (1, 2, 31, 128, 1025, 4096):
        T = R.cancelling(rng, 6, n)
        for t in range(T.shape[0]):
            exact = sum((Fraction(v) for v in T[t].tolist()), Fraction(0))
            for s in orders(rng, T[t]):
                assert abs(Fraction(s) - exact) <= Fraction(R.gamma(n - 1)) * sum(Fraction(abs(v)) for v in T[t].tolist())
                assert R.sum_within_bound(s, T[t])
        got = np.array([orders(rng, T[t])[-1] for t in range(T.shape[0])])
        assert R.sums_within_bound(got, T).all()
    # heavy cancellation: the sums are many orders of magnitude below sum |x|
    T = R.cancelling(rng, 4, 4096)
    assert np.all(np.abs([math.fsum(r.tolist()) for r in T]) < 1e-3 * np.abs(T).sum(axis=1))


@pytest.mark.parametrize("rowmajor", [False, True])
def test_planted_sum_errors_are_rejected(rowmajor):
    rng = np.random.default_rng(3 + rowmajor)
    r, c = 257, 1025
    for data in ("int", "cancelling"):
        a = rng.integers(-2 ** 20, 2 ** 20, (r, c)).astype(np.float64) if data == "int" else R.cancelling(rng, r, c)
        ds = {(0, 0): block(a[:, :600], rowmajor), (0, 1): block(a[:, 600:], not rowmajor)}
        T = R.lines("row", ds)[(0, 0)]
        assert np.array_equal(T, a)
        good = np.array([math.fsum(x.tolist()) for x in T])
        assert R.sums_within_bound(good, T).all()
        big = np.argmax(np.abs(T), axis=1)
        dropped = good - T[np.arange(r), big]
        twice = good + T[np.arange(r), big]
        # every row of block (0, 0) read with the other layout's stride: element (t, j) taken from values[t * c0 + j] (or
        # values[t + r * j]), i.e. the column-major / row-major image mixed up
        m = ds[(0, 0)]
        wrong = O.DenseMatrix(m.numRows, m.numCols, m.values, not m.isTransposed)
        Tw = R.lines("row", {(0, 0): wrong, (0, 1): ds[(0, 1)]})[(0, 0)]
        strided = np.array([math.fsum(x.tolist()) for x in Tw])
        for bad in (dropped, twice, strided):
            assert not R.sums_within_bound(bad, T).any()
            if data == "int":
                assert not np.any(bad == R.int_sums(T))
        assert not R.sum_within_bound(dropped[0], T[0]) and not R.sum_within_bound(twice[0], T[0])


def test_lines_match_the_oracle_aggregates():
    rng = np.random.default_rng(5)
    hs, ws = [31, 128, 1], [127, 1, 257]
    ds = {(i, j): block(rng.integers(-99, 99, (h, w)).astype(np.float64), (i + j) % 2 == 1)
          for i, h in enumerate(hs) for j, w in enumerate(ws)}
    for op, fn in (("row", O.row_sum), ("col", O.col_sum)):
        want = fn(ds, sum(hs), sum(ws))
        got = {k: R.int_sums(T) for k, T in R.lines(op, ds).items()}
        assert sorted(got) == sorted(want)
        assert all(np.array_equal(got[k], want[k].values) for k in want)
    (T,) = R.lines("sum", ds).values()
    assert R.int_sums(T)[0] == O.total_sum(ds, sum(hs), sum(ws))[(0, 0)].values[0]
    sq = {(i, j): block(rng.integers(-99, 99, (n, n)).astype(np.float64), i == 1) for i, n in enumerate([31, 128])
          for j in range(2) if i == j}
    (T,) = R.lines("trace", sq).values()
    assert T.shape == (1, 159) and R.int_sums(T)[0] == O.trace(sq, 159, 159)[(0, 0)].values[0]


def test_sum_classes():
    M = R.DBL_MAX
    assert R.sum_class([1.0, NAN]) == "nan" and R.sum_class([INF, -INF, 1.0]) == "nan"
    assert R.sum_class([INF, -1e300, -1e300]) == "+inf" and R.sum_class([-INF, 5.0]) == "-inf"
    assert R.sum_class([M, M, -1.0]) == "+inf" and R.sum_class([-M, -M * 0.75]) == "-inf"
    assert R.sum_class([1e308, 1e307, -5.0, TINY]) == "finite"
    for order_dependent in ([M, M, -M], [INF, -M, -M], [M, -M * 0.5, -M * 0.75]):
        with pytest.raises(ValueError):
            R.sum_class(order_dependent)
    assert R.sum_within_bound(INF, [M, M]) and not R.sum_within_bound(M, [M, M])
    assert R.sum_within_bound(0.0, [-0.0, -0.0]) and not R.sum_within_bound(-0.0, [-0.0, -0.0])
    assert R.sum_within_bound(0.0, [3.5, -3.5]) and not R.sum_within_bound(-0.0, [3.5, -3.5])
    assert R.sum_within_bound(3 * TINY, [TINY, TINY, TINY]) and not R.sum_within_bound(2 * TINY, [TINY, TINY, TINY])
    got = np.array([NAN, INF, 0.0, 1.0])
    T = np.array([[NAN, 1.0], [INF, 2.0], [0.0, -0.0], [0.5, 0.5]])
    assert R.sums_within_bound(got, T).all()
    assert not R.sums_within_bound(got[::-1], T).any()


def test_fma_rank_one_is_rejected():
    """x = y = 1 + 2^-30, a = -(1 + 2^-29): a + (x y) rounds x y to 1 + 2^-29 and gives 0.0; one fused rounding gives 2^-60."""
    x = 1.0 + 2.0 ** -30
    a = -(1.0 + 2.0 ** -29)
    fused = float(Fraction(a) + Fraction(x) * Fraction(x))
    assert fused == 2.0 ** -60
    A = O.DenseMatrix(1, 1, [a])
    v = O.DenseMatrix(1, 1, [x])
    want = O.rankOneAdd(A, v, v, compat_bugs=False).values
    assert same(want, [0.0]) and not same(want, [fused])
    # over a whole block: the two-rounding reference is numpy's a + outer(x, y); a fused result differs in many entries
    rng = np.random.default_rng(6)
    n = 64
    a = rng.standard_normal((n, n))
    xv, yv = rng.standard_normal(n), rng.standard_normal(n)
    want = O.rankOneAdd(block(a, True), block(xv.reshape(n, 1), False), block(yv.reshape(n, 1), False), compat_bugs=False)
    assert np.array_equal(R.dense_array(want), a + np.multiply.outer(xv, yv))
    fused = np.array([[float(Fraction(a[i, j]) + Fraction(xv[i]) * Fraction(yv[j])) for j in range(n)] for i in range(n)])
    assert np.count_nonzero(fused != R.dense_array(want)) > n


def test_java_pow_special_values():
    for x, p, want in R.SPECIAL:
        assert same([R.java_pow(x, p)], [want]), (x, p)
    # C's pow (Python's math.pow) gives 1.0 on the first five: rejected
    for x, p, want in R.SPECIAL[:5]:
        assert math.pow(x, p) == 1.0 and not same([math.pow(x, p)], [R.java_pow(x, p)])


def test_java_pow_is_correctly_rounded():
    rng = np.random.default_rng(7)
    xs = np.concatenate([rng.uniform(0, 4, 40), 2.0 ** rng.uniform(-1070, 1020, 40)])
    for p in (-1.3, 3.0, -2.0, 0.25, 1.0 / 3.0, 7.5, -0.5, 2.0, 0.5):
        for x in xs.tolist():
            got = R.java_pow(x, p)
            if p == 2.0:
                assert got == x * x
            elif p == 0.5:
                assert got == math.sqrt(x)
            else:
                exact = mp_pow(x, p)
                if math.isfinite(got) and got > 2.0 ** -1022:
                    # |got - x^p| <= ulp/2, and no other double is closer
                    assert abs(exact - Fraction(got)) <= Fraction(math.ulp(got)) / 2, (x, p)
    assert R.ulp_distance([1.0, 0.0, -TINY, INF], [np.nextafter(1.0, 2.0), -0.0, TINY, R.DBL_MAX]).tolist() == [1, 0, 2, 1]


def mp_pow(x, p):
    import mpmath
    with mpmath.workprec(300):
        y = mpmath.power(mpmath.mpf(x), mpmath.mpf(p))
        m, e = mpmath.frexp(y)
        return Fraction(int(mpmath.nint(m * mpmath.mpf(2) ** 280))) * Fraction(2) ** (int(e) - 280)


def test_oracle_matrix_pow_is_java_pow():
    xs = sorted({x for x, _, _ in R.SPECIAL} | {0.5, -0.5, 3.0, -3.0}, key=repr)
    ps = sorted({p for _, p, _ in R.SPECIAL}, key=repr)
    for p in ps:
        got = O.matrixPow(O.DenseMatrix(len(xs), 1, np.array(xs)), p).values
        want = [R.java_pow(x, p) for x in xs]
        special = [x == 0.0 or not math.isfinite(x) or abs(x) == 1.0 or not math.isfinite(p) or p in (0.0, 1.0) or
                   not math.isfinite(w) or w == 0.0 for x, w in zip(xs, want)]
        for x, g, w, sp in zip(xs, got, want, special):
            if sp:
                assert same([g], [w]), (x, p, g, w)
            else:
                assert R.ulp_distance([g], [w])[0] <= 1, (x, p, g, w)

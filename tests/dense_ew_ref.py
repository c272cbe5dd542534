"""Exact references for the dense element-wise, scalar, slicing and aggregate kernels (ew.cu), in plain Python: fractions,
math.fsum and mpmath.

  1. add / multiply / divide, scalar add / multiply, power(2), power(0.5), copies, project / selection and the rank-one update
     a + (x y) are single IEEE operations per element (two for the rank-one update, each rounded on its own).  numpy's float64
     operations do not contract, so the oracle gives the bits the kernels must give.
  2. rowSum / colSum / sum / trace: an output entry is the sum of its terms, gathered over every block of its line.  The dense
     kernels add with fp64 atomics in no fixed order (DESIGN section 4.5.4), so a finite result is held to the bound of every
     summation order (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., section 4.2):
         |s_hat - s| <= gamma_(n-1) sum |x_i|,   gamma_k = k u / (1 - k u),   u = 2^-53,   n terms,
     provided no partial sum can overflow.  Every sum starts at +0.0, so an exactly zero sum is +0.0.  Integer-valued terms whose
     absolute sum stays below 2^53 are added exactly in every order; their sums are compared bit for bit (int_sums).
  3. power with other exponents: java.lang.Math.pow (java_pow), whose special cases differ from C's pow (pow(+-1, +-inf) and
     pow(1, NaN) are NaN), the other values correctly rounded from mpmath.
"""
import math
from fractions import Fraction

import mpmath
import numpy as np

U = 2.0 ** -53
DBL_MAX = np.finfo(np.float64).max


def dense_array(m):
    """The numRows x numCols array of a dense block (isTransposed: values are row-major)."""
    v = np.asarray(m.values, dtype=np.float64)
    return v.reshape(m.numRows, m.numCols) if m.isTransposed else v.reshape(m.numCols, m.numRows).T


def lines(op, ds):
    """{output key: T} for op in 'row', 'col', 'sum', 'trace' over a dict of dense blocks: row t of T holds the terms of output
    entry t, gathered over every block of its line in ascending block index."""
    by_key = {}
    for (rid, cid), m in sorted(ds.items()):
        if op == "trace" and rid != cid:
            continue
        a = dense_array(m)
        if op == "row":
            by_key.setdefault((rid, 0), []).append(a)
        elif op == "col":
            by_key.setdefault((0, cid), []).append(a.T)
        elif op == "sum":
            by_key.setdefault((0, 0), []).append(a.reshape(1, -1))
        else:
            by_key.setdefault((0, 0), []).append(np.diag(a).reshape(1, -1))
    return {k: np.concatenate(v, axis=1) for k, v in by_key.items()}


def gamma(k):
    return k * U / (1.0 - k * U)


def int_sums(T):
    """The exact sums of the rows of T, all of whose terms are integers with sum |x| < 2^53: any order gives these bits."""
    assert np.all(T == np.round(T)), "int_sums needs integer-valued terms"
    Ti = T.astype(np.int64)
    assert np.all(np.abs(Ti).sum(axis=1) < 2 ** 53), "int_sums needs sum |x| < 2^53"
    return Ti.sum(axis=1).astype(np.float64)


def _abs_sum(x):
    try:
        return math.fsum(np.abs(x).tolist())
    except OverflowError:
        return math.inf


def sum_class(x):
    """'nan', '+inf', '-inf' or 'finite': the class every summation order of the terms x gives.  Raises ValueError when the class
    depends on the order (a partial sum may overflow in some orders and not in others)."""
    x = np.asarray(x, dtype=np.float64)
    pinf, ninf = bool(np.isposinf(x).any()), bool(np.isneginf(x).any())
    if np.isnan(x).any() or (pinf and ninf):
        return "nan"
    f = x[np.isfinite(x)]
    slack = 1.0 + gamma(max(x.size, 1))
    pos = _abs_sum(f[f > 0]) * slack   # bounds every partial sum of the finite terms, in every order
    neg = _abs_sum(f[f < 0]) * slack
    if pinf or ninf:
        if (neg if pinf else pos) < DBL_MAX:  # no partial sum can overflow the other way
            return "+inf" if pinf else "-inf"
        raise ValueError("order-dependent: an infinity meets finite terms that may overflow to the other one")
    if pos < DBL_MAX and neg < DBL_MAX and _abs_sum(f) * slack < DBL_MAX:
        return "finite"
    s = sum((Fraction(float(v)) for v in f), Fraction(0))
    tol = Fraction(gamma(max(x.size - 1, 0))) * sum((Fraction(abs(float(v))) for v in f), Fraction(0))
    if neg < DBL_MAX and s - tol > Fraction(DBL_MAX):
        return "+inf"  # no partial goes below -DBL_MAX, and a sum that never overflowed would be above DBL_MAX
    if pos < DBL_MAX and s + tol < -Fraction(DBL_MAX):
        return "-inf"
    raise ValueError("order-dependent: partial sums may overflow")


def sum_within_bound(got, x):
    """True when got is a sum of the terms x in some order: the class of sum_class, and for a finite class
    |got - s| <= gamma_(n-1) sum |x| (s the exact sum), with +0.0 for an exactly zero sum."""
    got = float(got)
    cls = sum_class(x)
    if cls == "nan":
        return math.isnan(got)
    if cls != "finite":
        return got == (math.inf if cls == "+inf" else -math.inf)
    if not math.isfinite(got):
        return False
    if got == 0.0 and math.copysign(1.0, got) < 0:
        return False  # sums start at +0.0 and doubles add without underflow: a zero sum is +0.0
    xs = np.asarray(x, dtype=np.float64).tolist()
    fs = math.fsum(xs)  # the correctly rounded sum
    # |got - s| <= |got - fs| + |fs - s| and |fs - s| <= ulp(fs) / 2: that half ulp is allowed on top of the bound, and a
    # relative 2^-40 for the rounding of the bound itself
    allowed = Fraction(gamma(max(len(xs) - 1, 0))) * Fraction(_abs_sum(xs)) * (1 + Fraction(1, 2 ** 40)) + Fraction(math.ulp(fs)) / 2
    return abs(Fraction(got) - Fraction(fs)) <= allowed


def sums_within_bound(got, T):
    """sum_within_bound(got[t], T[t]) for every row t of T, as a boolean array.  Rows of finite terms that cannot overflow take a
    vectorised path: numpy's sum of |x| times (1 + gamma_n) bounds sum |x| from above (a sum of non-negative doubles is within
    gamma_(n-1) of the exact one), and the half ulp and the 2^-40 of sum_within_bound absorb the rounding of |got - fsum|."""
    got = np.asarray(got, dtype=np.float64).reshape(-1)
    T = np.asarray(T, dtype=np.float64)
    assert T.ndim == 2 and got.size == T.shape[0]
    n = T.shape[1]
    with np.errstate(over="ignore", invalid="ignore"):
        abs_hi = np.abs(T).sum(axis=1) * (1.0 + gamma(n))
    fast = np.isfinite(T).all(axis=1) & (abs_hi * (1.0 + gamma(n)) < DBL_MAX)
    ok = np.zeros(T.shape[0], dtype=bool)
    for t in np.flatnonzero(~fast):
        ok[t] = sum_within_bound(got[t], T[t])
    idx = np.flatnonzero(fast)
    if idx.size:
        fs = np.array([math.fsum(T[t].tolist()) for t in idx])
        g = got[idx]
        allowed = gamma(max(n - 1, 0)) * abs_hi[idx] * (1.0 + 2.0 ** -40) + np.spacing(np.abs(fs)) / 2
        with np.errstate(invalid="ignore"):
            ok[idx] = np.isfinite(g) & (np.abs(g - fs) <= allowed) & ~((g == 0.0) & np.signbit(g))
    return ok


def ordered(v):
    """float64 values as integers that are consecutive for consecutive doubles (-0.0 and +0.0 both map to 0)."""
    i = np.asarray(v, dtype=np.float64).reshape(-1).view(np.int64).astype(object)
    return [int(k) if k >= 0 else -(int(k) & 0x7FFFFFFFFFFFFFFF) for k in i]


def ulp_distance(a, b):
    """Number of doubles between a and b (elementwise, finite or infinite, not NaN)."""
    return np.array([abs(p - q) for p, q in zip(ordered(a), ordered(b))], dtype=object)


def bits(v):
    """float64 values as int64 bits, every NaN mapped to one pattern (payloads may differ)."""
    v = np.array(v, dtype=np.float64, copy=True).reshape(-1)
    v[np.isnan(v)] = np.nan
    return v.view(np.int64)


def _odd_int(p):
    return math.isfinite(p) and p == math.floor(p) and math.fmod(p, 2.0) != 0.0


def _round_to_double(y):
    """The double nearest to the positive mpf y (ties to even), with subnormals and overflow."""
    if y >= mpmath.mpf(2) ** 1024 - mpmath.mpf(2) ** 970:
        return math.inf
    if y < mpmath.mpf(2) ** -1022:
        return float(mpmath.nint(y * mpmath.mpf(2) ** 1074)) * 2.0 ** -1074
    with mpmath.workprec(53):
        r = +y  # rounds to nearest at 53 bits
    return float(r)


def java_pow(x, p):
    """java.lang.Math.pow(x, p): the special cases of its specification, and the correctly rounded x^p otherwise."""
    x, p = float(x), float(p)
    if p == 0.0:
        return 1.0
    if p == 1.0:
        return x
    if math.isnan(p) or math.isnan(x):
        return math.nan
    if math.isinf(p):
        ax = abs(x)
        if ax == 1.0:
            return math.nan
        return math.inf if (ax > 1.0) == (p > 0.0) else 0.0
    odd = _odd_int(p)
    if x == 0.0 or math.isinf(x):
        mag = math.inf if (x != 0.0) == (p > 0.0) else 0.0
        return math.copysign(mag, x) if odd else mag
    if x < 0.0:
        if p != math.floor(p):
            return math.nan
        r = java_pow(-x, p)
        return -r if odd else r
    with mpmath.workprec(256):
        y = mpmath.power(mpmath.mpf(x), mpmath.mpf(p))
    return _round_to_double(y)


def cancelling(rng, rows, cols):
    """Full 53-bit mantissas over 40 binades, every other term close to the negation of its neighbour: |sum| << sum |x|."""
    a = rng.uniform(-1.0, 1.0, (rows, cols)) * 2.0 ** rng.integers(0, 40, (rows, cols))
    a[:, 1::2] = -a[:, 0:cols - 1:2] * (1.0 + rng.uniform(-2.0 ** -20, 2.0 ** -20, (rows, cols // 2)))
    return a


NAN, INF, TINY = math.nan, math.inf, 2.0 ** -1074

# (x, p, java.lang.Math.pow(x, p)) from the special cases of its specification; the first five differ from C's pow
SPECIAL = [
    (1.0, INF, NAN), (1.0, -INF, NAN), (-1.0, INF, NAN), (-1.0, -INF, NAN), (1.0, NAN, NAN),
    (NAN, 0.0, 1.0), (NAN, -0.0, 1.0), (2.0, 0.0, 1.0), (NAN, 1.0, NAN), (-0.0, 1.0, -0.0), (3.5, 1.0, 3.5),
    (2.0, NAN, NAN), (NAN, 2.0, NAN), (-1.0, NAN, NAN),
    (2.0, INF, INF), (0.5, -INF, INF), (-2.0, INF, INF), (2.0, -INF, 0.0), (0.5, INF, 0.0), (-0.5, INF, 0.0),
    (0.0, 2.5, 0.0), (INF, -2.5, 0.0), (0.0, -2.5, INF), (INF, 2.5, INF),
    (-0.0, 2.5, 0.0), (-0.0, 2.0, 0.0), (-INF, -2.5, 0.0), (-INF, -2.0, 0.0),
    (-0.0, 3.0, -0.0), (-INF, -3.0, -0.0),
    (-0.0, -2.5, INF), (-0.0, -2.0, INF), (-INF, 2.5, INF), (-INF, 2.0, INF),
    (-0.0, -3.0, -INF), (-INF, 3.0, -INF),
    (-2.0, 2.0, 4.0), (-2.0, 3.0, -8.0), (-2.0, 0.5, NAN), (-8.0, 1.0 / 3.0, NAN),
    (2.0, 1024.0, INF), (2.0, -1074.0, TINY), (2.0, -1075.0, 0.0), (-2.0, -1075.0, -0.0), (4.0, 0.5, 2.0), (-0.0, 0.5, 0.0),
    (-INF, 0.5, INF), (TINY, 0.5, 2.0 ** -537), (1e308, 2.0, INF),
]

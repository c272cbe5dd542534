"""CPU checks of tests/tf32_ref.py: the tf32 rounding, the exact-regime generators, the exact model against the exact reference,
the truncating simulation against the bound, and planted defects that the model or the bound must expose."""
from fractions import Fraction

import numpy as np
import pytest

from tests.exact_ref import exact_entries
from tests.tf32_ref import (CHUNK, mean, prepare, regime_ok, regime_operand, scale_exp, simulate_truncating, split, tf32_bound,
                            tf32_exact_model, to_tf32)

F = np.float32


@pytest.mark.parametrize("x,want", [
    (1.0, 1.0),
    (1 + 2.0 ** -11, 1 + 2.0 ** -10),                       # tie: away from zero
    (1 + 2.0 ** -11 - 2.0 ** -23, 1.0),                     # just below the tie
    (1 + 3 * 2.0 ** -11, 1 + 2 * 2.0 ** -10),               # tie at an odd tf32 mantissa: away from zero, not to even
    (-(1 + 2.0 ** -11), -(1 + 2.0 ** -10)),                 # negative tie
    (-(1 + 2.0 ** -11 - 2.0 ** -23), -1.0),
    (2 - 2.0 ** -11, 2.0),                                  # carry into the exponent
    (-(2 - 2.0 ** -11), -2.0),
    (2 - 2.0 ** -10, 2 - 2.0 ** -10),                       # already tf32
    (2.0 ** -126 * (1 + 2.0 ** -11), 2.0 ** -126 * (1 + 2.0 ** -10)),
    (0.0, 0.0),
])
def test_to_tf32_rounds_to_nearest_ties_away(x, want):
    got = to_tf32(np.array([x], dtype=F))
    assert got.dtype == F and got[0] == F(want), (x, float(got[0]), want)
    assert (got.view(np.uint32) & 0x1FFF == 0).all()


def test_split_is_exact_for_22_bit_values_and_within_2_22_otherwise():
    rng = np.random.default_rng(1)
    x = rng.uniform(-4, 4, 100000).astype(F)
    hi, lo = split(x)
    assert ((hi.view(np.uint32) & 0x1FFF) == 0).all() and ((lo.view(np.uint32) & 0x1FFF) == 0).all()
    err = np.abs(x.astype(np.float64) - hi - lo)
    assert (err <= 2.0 ** -22 * np.abs(x)).all()
    assert (err > 0).any()
    y = to_tf32(x) + to_tf32(x * F(2.0 ** -11))                # values hi + lo with two 11-bit parts
    y = y[np.abs(y) >= 2.0 ** -100]
    hy, ly = split(y)
    assert np.array_equal(hy.astype(np.float64) + ly, y.astype(np.float64))


def test_scale_exponent_puts_the_largest_magnitude_in_1_2():
    for mx in (1.0, 1.5, 2.0 - 2.0 ** -52, 1e-20, 1e20, 1e-300, 1e300, 2.0 ** -1074, np.finfo(np.float64).max):
        s = scale_exp(np.array([[mx, -mx / 3]]))
        assert 1.0 <= np.ldexp(mx, -s) < 2.0, mx
    assert scale_exp(np.zeros((2, 2))) == 0


def test_prepare_flushes_below_2_126():
    X = np.array([[1.0, 2.0 ** -127, -2.0 ** -126, 2.0 ** -149, 1 + 2.0 ** -30]])
    a, hi, lo = prepare(X, 0.0, 0)
    assert a[0].tolist() == [1.0, 0.0, -2.0 ** -126, 0.0, 1.0]
    a, hi, lo = prepare(np.array([[(1 + 2.0 ** -20) * 2.0 ** -110]]), 0.0, 0)   # hi = 2^-110, lo = 2^-130: flushed
    assert hi[0, 0] == F(2.0 ** -110) and lo[0, 0] == 0.0


# ---------------------------------------------------------------------------------------------------------------- regime
REGIME = [  # n, K, m, offset, exp
    (16, 64, 16, 0.0, 0),
    (16, 64, 16, 0.5, 0),
    (8, 2048, 16, 0.5, 3),
    (16, 4096, 8, 0.5, -40),
    (5, 2049, 7, 0.0, 0),
    (3, 4097, 6, 0.0, 700),
]


@pytest.mark.parametrize("n,K,m,offset,exp", REGIME)
def test_regime_generators_are_exact(n, K, m, offset, exp):
    rng = np.random.default_rng(n + K + m)
    A = regime_operand(rng, (n, K), density=0.4, offset=offset, exp=exp)
    B = regime_operand(rng, (K, m), density=0.4, offset=offset, exp=-exp)
    muA, muB = mean(A), mean(B)
    assert muA == np.ldexp(offset, exp) and muB == np.ldexp(offset, -exp)
    # the device's total, in any order, is exact: the n-parts cancel in pairs and all partial sums lie on a coarse grid
    assert float(np.sum(A[::-1])) == math_sum(A) and np.sum(np.sort(A, axis=None)) == math_sum(A)
    assert regime_ok(A, B, (muA, muB))
    assert scale_exp(A) == exp and scale_exp(B) == -exp
    a, hi, lo = prepare(A, muA, exp)
    assert set(np.unique(hi)) == {-1.0, 0.0, 1.0} and set(np.unique(lo)) == {-2.0 ** -12, 0.0, 2.0 ** -12}


def math_sum(X):
    return float(sum(Fraction(float(v)) for v in X.ravel()))


def model_against_exact(A, B, mu):
    """tf32_exact_model == exact(A B) - 2^(sA + sB) lo_A lo_B at every entry, both correctly rounded from exact values."""
    sA, sB = scale_exp(A), scale_exp(B)
    _, _, la = prepare(A, mu[0], sA)
    _, _, lb = prepare(B, mu[1], sB)
    n, m = A.shape[0], B.shape[1]
    pos = [(i, j) for i in range(n) for j in range(m)]
    ex = exact_entries(A, B, pos)
    ll = exact_entries(np.ldexp(la.astype(np.float64), sA), np.ldexp(lb.astype(np.float64), sB), pos)
    model = tf32_exact_model(A, B, mu)
    for (i, j), x, y in zip(pos, ex, ll):
        assert model[i, j] == float(x - y), (i, j, model[i, j], float(x - y))
    return model


@pytest.mark.parametrize("n,K,m,offset,exp", REGIME)
def test_model_equals_the_exact_reference(n, K, m, offset, exp):
    rng = np.random.default_rng(7 * n + K + m)
    A = regime_operand(rng, (n, K), density=0.4, offset=offset, exp=exp)
    B = regime_operand(rng, (K, m), density=0.4, offset=offset, exp=-exp)
    model_against_exact(A, B, (mean(A), mean(B)))
    if offset == 0.0:
        model_against_exact(A, B, (0.0, 0.0))                  # uncentred (absent blocks): the means stay 0


def test_model_rejects_data_outside_the_regime():
    rng = np.random.default_rng(3)
    A, B = rng.uniform(-1, 1, (4, 64)), rng.uniform(-1, 1, (64, 4))
    assert not regime_ok(A, B)
    with pytest.raises(AssertionError):
        tf32_exact_model(A, B)
    A, B = np.full((2, 2048), 1 - 2.0 ** -11), np.full((2048, 2), 1 - 2.0 ** -11)
    assert not regime_ok(A, B)                                 # 1 - 2^-11 is its own hi: hi hi' lies on the 2^-22 grid


# ---------------------------------------------------------------------------------------------------------------- bound
def bound_holds(A, B, mu, got):
    n, m = A.shape[0], B.shape[1]
    pos = [(i, j) for i in range(n) for j in range(m)]
    E = tf32_bound(A, B, mu)
    worst = 0.0
    for (i, j), x in zip(pos, exact_entries(A, B, pos)):
        err = abs(Fraction(float(got[i, j])) - x)
        assert err <= Fraction(float(E[i, j])), (i, j, float(err), E[i, j])
        worst = max(worst, float(err) / E[i, j])
    return worst


def cancelling(rng, n, K, m):
    """Rows (a, -a) against columns (b, b) with a tail of 2^-30: C is nearly 0, carried by the small terms."""
    A, B = rng.uniform(1, 2, (n, K)), rng.uniform(1, 2, (K, m))
    h = K // 2 - 4
    A[:, h:2 * h] = -A[:, :h]
    B[h:2 * h] = B[:h]
    A[:, 2 * h:] *= 2.0 ** -30
    return A, B


DATA = {
    "uniform": lambda rng, n, K, m: (rng.uniform(-1, 1, (n, K)), rng.uniform(-1, 1, (K, m))),
    "offset_1e6": lambda rng, n, K, m: (1e6 + rng.uniform(0, 1, (n, K)), 1e6 + rng.uniform(0, 1, (K, m))),
    "positive": lambda rng, n, K, m: (rng.uniform(0, 1, (n, K)), rng.uniform(0, 1, (K, m))),
    "cancelling": cancelling,
    "wide_range": lambda rng, n, K, m: (rng.uniform(-1, 1, (n, K)) * np.exp2(rng.integers(-60, 60, (n, K))),
                                        rng.uniform(-1, 1, (K, m)) * np.exp2(rng.integers(-60, 60, (K, m)))),
    "tiny": lambda rng, n, K, m: (1e-20 * rng.uniform(-1, 1, (n, K)), 1e-20 * rng.uniform(-1, 1, (K, m))),
    "huge": lambda rng, n, K, m: (1e150 * rng.uniform(-1, 1, (n, K)), 1e150 * rng.uniform(-1, 1, (K, m))),
}


@pytest.mark.parametrize("K", [100, 2100])
@pytest.mark.parametrize("centred", [True, False])
@pytest.mark.parametrize("data", sorted(DATA))
def test_truncating_accumulation_stays_within_the_bound(data, centred, K):
    rng = np.random.default_rng(len(data) + K)
    n, m = 4, 5
    A, B = DATA[data](rng, n, K, m)
    mu = (mean(A), mean(B)) if centred else (0.0, 0.0)
    got = simulate_truncating(A, B, mu)
    assert np.isfinite(got).all()
    worst = bound_holds(A, B, mu, got)
    assert worst < 1.0


def test_the_bound_is_not_vacuous():
    """On positive data (the worst case for a truncating accumulator) the bound stays far below |A||B|."""
    rng = np.random.default_rng(5)
    A, B = DATA["positive"](rng, 4, 2100, 5)
    E = tf32_bound(A, B, (mean(A), mean(B)))
    U = np.abs(A) @ np.abs(B)
    assert (E < 1e-2 * U).all() and (E > 1e-4 * U).all()


def test_simulation_truncates():
    """Uncentred positive data: every addition truncated gives a one-sided error (the bias centring removes)."""
    rng = np.random.default_rng(6)
    A, B = DATA["positive"](rng, 4, 2100, 5)
    got = simulate_truncating(A, B)
    exact = np.array([[float(x) for x in exact_entries(A, B, [(i, j)])] for i in range(4) for j in range(5)]).reshape(4, 5)
    assert (got < exact).all()


# ---------------------------------------------------------------------------------------------------------------- planted
def row_major_read_column_major(A, blk):
    """Block (0, 0) of A stored row-major but read with the column-major stride."""
    A = A.copy()
    r, c = min(blk, A.shape[0]), min(blk, A.shape[1])
    A[:r, :c] = A[:r, :c].ravel(order="C").reshape((r, c), order="F")
    return A


@pytest.mark.parametrize("plant", ["drop_lo_hi", "drop_hi_lo", "padded_mean", "corr_every_chunk", "lost_chunk", "scale_off_by_one",
                                   "row_major_stride"])
def test_planted_defects_change_the_model(plant):
    rng = np.random.default_rng(9)
    n, K, m = 8, 4096, 8                                       # two chunks; M K and K N powers of two; Mpad != M
    A = regime_operand(rng, (n, K), density=0.4, offset=0.5, exp=2)
    B = regime_operand(rng, (K, m), density=0.4, offset=0.5, exp=-1)
    mu = (mean(A), mean(B))
    model = tf32_exact_model(A, B, mu)
    if plant == "row_major_stride":
        A2 = row_major_read_column_major(A, 6)
        planted = tf32_exact_model(A2, B, (mean(A2), mu[1]))
    elif plant == "padded_mean":                               # the centred values leave the regime: replay a truncating device
        planted = simulate_truncating(A, B, (mu[0] * (n * K) / (128 * K), mu[1] * (K * m) / (K * 256)))
    else:
        planted = tf32_exact_model(A, B, mu, plant=plant)
    assert (model.view(np.int64) != planted.view(np.int64)).any(), plant
    assert K > CHUNK

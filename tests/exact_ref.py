"""Exact reference for fp64 matrix products, and the element-wise error bound of the Ozaki-II multiply.

fp64 values are dyadic rationals, so a dot product of two fp64 vectors is an exact integer times a power of two: every
element is split into a 53-bit Python integer and an exponent (np.frexp, which normalises sub-normals), the products are
summed as big integers over the smallest exponent present, and the result is returned as a Fraction.  float(Fraction) is
correctly rounded, so round_to_double() of an exact entry is THE fp64 value of that entry of the product."""
import math
import os
import re
from fractions import Fraction

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _split(v):
    """1-D fp64 array -> (53-bit signed integer mantissas, exponents) with v = mant * 2^exp exactly (zeros: mant = 0)."""
    v = np.asarray(v, dtype=np.float64)
    assert np.all(np.isfinite(v)), "exact reference of non-finite data"
    m, e = np.frexp(v)                                     # |m| in [0.5, 1), also for sub-normal v
    return np.ldexp(m, 53).astype(np.int64).tolist(), (e.astype(np.int64) - 53).tolist()


def exact_dot(a, b):
    """sum_k a_k b_k of two fp64 vectors as an exact Fraction."""
    ma, ea = _split(a)
    mb, eb = _split(b)
    terms = [(x * y, p + q) for x, p, y, q in zip(ma, ea, mb, eb) if x and y]
    if not terms:
        return Fraction(0)
    emin = min(e for _, e in terms)
    total = sum(t << (e - emin) for t, e in terms)
    return Fraction(total) * Fraction(2) ** emin


def exact_entries(A, B, ij_pairs):
    """Exact (A B)[i, j] for each (i, j) of ij_pairs, as Fractions."""
    A, B = np.asarray(A, dtype=np.float64), np.asarray(B, dtype=np.float64)
    assert A.ndim == 2 and B.ndim == 2 and A.shape[1] == B.shape[0]
    return [exact_dot(A[i, :], B[:, j]) for i, j in ij_pairs]


def round_to_double(x):
    """The fp64 value nearest to the Fraction x (ties to even); +-inf beyond the fp64 range."""
    try:
        return float(x)
    except OverflowError:
        return math.inf if x > 0 else -math.inf


# ---- the moduli and the operand width alpha, from the documented rule (never read off the device)
_SRC = open(os.path.join(ROOT, "matrel_b200", "csrc", "gemm_ozaki.cu")).read()
MODULI = [int(x) for x in re.search(r"kCrtModuli\[CRT_MAX_T\] = \{([^}]*)\}", _SRC).group(1).split(",")]
T_MIN, T_MAX = int(re.search(r"CRT_MIN_T = (\d+)", _SRC).group(1)), int(re.search(r"CRT_MAX_T = (\d+)", _SRC).group(1))


def ceil_log2(K):
    lg = 0
    while (1 << lg) < K:
        lg += 1
    return lg


def alpha_of(T, K):
    """alpha = floor((floor(log2 P) - 1 - ceil(log2 K)) / 2), at most 62 (the rule test_crt_math_cpu.py checks)."""
    P = math.prod(MODULI[:T])
    return min(62, (P.bit_length() - 1 - 1 - ceil_log2(K)) // 2)


def moduli_for(K, requested=0):
    """crt_moduli = 0: the smallest count with alpha >= 54 - ceil(lg K / 2); else the requested count, clamped."""
    if requested > 0:
        return min(T_MAX, max(T_MIN, requested))
    want = 54 - (ceil_log2(K) + 1) // 2
    return next((t for t in range(T_MIN, T_MAX + 1) if alpha_of(t, K) >= want), T_MAX)


def oz2_bound(A, B, alpha, C=None):
    """Element-wise bound of |got - exact| for the Ozaki-II product of A (n x K) and B (K x m).

    Row i of A is rounded to multiples of 2^(e_i - alpha) with 2^e_i <= 2 rowmax_i, so |da_ik| <= 2^-alpha rowmax_i; columns
    of B likewise.  The integer product of the rounded operands is exact, hence
        |err_ij| <= sum_k |da_ik| |b_kj| + |a_ik| |db_kj| + |da_ik| |db_kj|
                 <= 2^-alpha (rowmax_i sum_k |b_kj| + colmax_j sum_k |a_ik|) (1 + K 2^-alpha)
    plus the rounding of the reconstructed integer to fp64: below one ulp (the chunked Horner sum of crt_kernel rounds at most
    twice), i.e. 2^-52 |C_ij|, and four units of the smallest sub-normal for results scaled into the sub-normal range.
    Elements handled as exact outliers contribute no operand error, so the bound also holds under the range guard.
    C: the exact product or anything close to it (numpy's A @ B); left out, the rounding term uses |A||B| >= |C|."""
    A, B = np.asarray(A, dtype=np.float64), np.asarray(B, dtype=np.float64)
    K = A.shape[1]
    with np.errstate(over="ignore", invalid="ignore"):
        absA, absB = np.abs(A), np.abs(B)
        rowmax, colmax = absA.max(axis=1, initial=0.0), absB.max(axis=0, initial=0.0)
        u = 2.0 ** -alpha
        # extended precision for the sums: the bound itself must not overflow for operands near the top of the fp64 range
        ld = np.longdouble
        op = rowmax.astype(ld)[:, None] * absB.astype(ld).sum(axis=0)[None, :] + absA.astype(ld).sum(axis=1)[:, None] * colmax.astype(ld)[None, :]
        op = np.minimum(op * ld(u * (1.0 + K * u)), ld(np.finfo(np.float64).max)).astype(np.float64)
        mag = np.abs(C) if C is not None else absA @ absB
        return op + 2.0 ** -52 * mag + 4 * 2.0 ** -1074


def fp64_dot_bound(A, B):
    """Classical bound of a length-K fp64 dot product in any summation order: K 2^-53 |A||B| (first order, with 1 % slack), plus
    one unit of the smallest sub-normal per term for products and partial sums that underflow."""
    A, B = np.asarray(A, dtype=np.float64), np.asarray(B, dtype=np.float64)
    with np.errstate(over="ignore"):
        return 1.01 * A.shape[1] * 2.0 ** -53 * (np.abs(A) @ np.abs(B)) + (A.shape[1] + 4) * 2.0 ** -1074

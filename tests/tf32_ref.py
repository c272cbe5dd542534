"""Reference, exact model and error bound of the fp32 multiply on wgmma tf32 (gemm_algo 3, DESIGN section 4.3).

The device centres each operand by its mean mu (when the blocks cover it completely), scales it by 2^-s with s = ilogb(max |a|),
rounds a' = fl32((a - mu) 2^-s) (values below 2^-126 flushed), splits hi = tf32(a'), lo = tf32(a' - hi), and sums
lo hi' + hi lo' + hi hi' in fp32 on the tensor core, one 2048-deep K chunk at a time.  Chunk sums are scaled by 2^(sA + sB) and
re-accumulated in fp64; the first chunk also adds the fp64 mean corrections muB (A'1)_i + K muA muB + muA (1^T B')_j.

tf32_exact_model is that arithmetic where it is exact: on operands built by regime_operand every partial sum of the fp32
accumulator is representable whatever the order, so the device result is defined without any assumption about how the tensor
core accumulates, and equals exact(A B) - 2^(sA+sB) lo_A lo_B.  tf32_bound is the element-wise bound elsewhere; it assumes the
fp32 accumulator truncates each addition by at most 2^-23 of the running magnitude (checked on the GPU by
tests/test_gpu_tf32_edges.py).  simulate_truncating replays a truncating accumulator in the kernel's order (small sizes only)."""
import math

import numpy as np

CHUNK = 2048            # K elements per fp32 chunk (64 stages of 32)
FLUSH = 2.0 ** -126     # a' and lo below this are zero
LO_GRID = 2.0 ** -12


def to_tf32(x):
    """cvt.rna.tf32.f32: round the 13 dropped mantissa bits to nearest, ties away from zero (finite fp32 input)."""
    u = np.asarray(x, dtype=np.float32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def split(a):
    """a: fp32 array -> (hi, lo) = (tf32(a), tf32(a - hi)); a - hi is exact in fp32."""
    a = np.asarray(a, dtype=np.float32)
    hi = to_tf32(a)
    return hi, to_tf32(a - hi)


def scale_exp(X):
    """s with max |X| 2^-s in [1, 2); 0 for an all-zero operand."""
    mx = float(np.max(np.abs(X), initial=0.0))
    return math.frexp(mx)[1] - 1 if mx > 0 else 0


def mean(X, count=None):
    """The operand mean as the device forms it: total * (1 / count), count = the operand's extent (default X.size).  The device's
    total is summed in a fixed order of its own; this one is exact, so the two agree whenever the total is exact in fp64."""
    count = X.size if count is None else count
    return math.fsum(np.asarray(X, dtype=np.float64).ravel()) * (1.0 / float(count))


def prepare(X, mu, s):
    """fp64 operand -> (a', hi, lo) as fp32 arrays: a' = fl32((X - mu) 2^-s), flushed below 2^-126, lo flushed likewise."""
    a = np.ldexp(np.asarray(X, dtype=np.float64) - mu, -s).astype(np.float32)
    a[np.abs(a) < FLUSH] = 0.0
    hi, lo = split(a)
    lo[np.abs(lo) < FLUSH] = 0.0
    return a, hi, lo


# ---------------------------------------------------------------------------------------------------------------- exact regime
def regime_operand(rng, shape, density=0.5, offset=0.0, exp=0):
    """Entries (n1 (1 + n2 2^-12) + offset) 2^exp with n1, n2 in {-1, 0, 1} (non-zero with probability `density`), the n-part
    summing to exactly 0: half of the entries are the negatives of the other half, in random places.  Centred by the mean
    (= offset 2^exp exactly when the entry count is a power of two) and scaled, every value is hi + lo with hi = n1 and
    lo = n1 n2 2^-12 (1 - 2^-12 rounds to 1 in tf32: a tie, away from zero; 1 + 2^-11 would not split so)."""
    size = int(np.prod(shape))
    h = size // 2
    n1 = rng.choice([-1.0, 1.0], h) * (rng.random(h) < density)
    n2 = rng.choice([-1.0, 1.0], h) * (rng.random(h) < density)
    half = n1 * (1 + n2 * LO_GRID)
    flat = np.zeros(size)
    perm = rng.permutation(size)
    flat[perm[:h]], flat[perm[h:2 * h]] = half, -half
    return np.ldexp(flat.reshape(shape) + offset, exp)


def regime_ok(A, B, mu=(0.0, 0.0)):
    """True when every partial sum of the fp32 accumulator is exact for A B, in any order and under any chunking: the scaled
    centred values are hi + lo with hi in {-1, 0, 1} and lo in {0, +-2^-12} (so every product lies on the 2^-12 grid), and
    for each (i, j) the sum of |lo hi'| + |hi lo'| + |hi hi'| over all of K is at most 2^11 (23 bits of that grid)."""
    a, ha, la = prepare(A, mu[0], scale_exp(A))
    b, hb, lb = prepare(B, mu[1], scale_exp(B))
    for x, hx, lx in ((a, ha, la), (b, hb, lb)):
        if not (np.isin(hx, (-1.0, 0.0, 1.0)).all() and np.isin(lx, (-LO_GRID, 0.0, LO_GRID)).all() and np.array_equal(hx + lx, x)):
            return False
    mag = np.abs(la).astype(np.float64) @ np.abs(hb) + np.abs(ha).astype(np.float64) @ (np.abs(lb) + np.abs(hb))
    return bool((mag <= 2.0 ** 11).all())


def _corrections(a, sA, b, sB, mu, K):
    """Row and column corrections in fp64: muB (A'1)_i + K muA muB and muA (1^T B')_j, A' = a' 2^sA unscaled (exact in fp64)."""
    rows = np.ldexp(a.astype(np.float64), sA).sum(axis=1)
    cols = np.ldexp(b.astype(np.float64), sB).sum(axis=0)
    return mu[1] * rows + K * mu[0] * mu[1], mu[0] * cols


def tf32_exact_model(A, B, mu=(0.0, 0.0), plant=None):
    """The device result of A (n x K) times B (K x m), bit for bit, for operands in the exact regime (regime_ok); mu = the
    operand means the device uses (0 when the blocks do not cover an operand).  `plant` injects a known defect (tests only):
    'drop_lo_hi', 'drop_hi_lo', 'corr_every_chunk', 'lost_chunk', 'scale_off_by_one' (2^(sA + sB + 1) in the epilogue)."""
    A, B = np.asarray(A, dtype=np.float64), np.asarray(B, dtype=np.float64)
    n, K = A.shape
    m = B.shape[1]
    sA, sB = scale_exp(A), scale_exp(B)
    a, ha, la = prepare(A, mu[0], sA)
    b, hb, lb = prepare(B, mu[1], sB)
    rc, cc = _corrections(a, sA, b, sB, mu, K)
    corr = rc[:, None] + cc[None, :]
    e = sA + sB + (1 if plant == "scale_off_by_one" else 0)
    C = None
    for t, k0 in enumerate(range(0, K, CHUNK)):
        if plant == "lost_chunk" and t == 1:
            continue
        ks = slice(k0, min(K, k0 + CHUNK))
        f = lambda x, y: x[:, ks].astype(np.float64) @ y[ks].astype(np.float64)  # noqa: E731
        acc = (0 if plant == "drop_lo_hi" else f(la, hb)) + (0 if plant == "drop_hi_lo" else f(ha, lb)) + f(ha, hb)
        assert np.array_equal(np.asarray(acc, dtype=np.float32), acc), "not in the exact regime"
        term = np.ldexp(acc, e)
        if C is None or plant == "corr_every_chunk":
            term = term + corr
        C = term if C is None else C + term
    if C is None:                                    # a lost first and only chunk
        C = np.zeros((n, m))
    return C


# ---------------------------------------------------------------------------------------------------------------- the bound
def tf32_bound(A, B, mu=(0.0, 0.0)):
    """Element-wise bound of |device - exact(A B)| (DESIGN section 4.3), from magnitudes only.  With U_ij = sum_k (|a_ik| + |muA|)
    (|b_kj| + |muB|) >= sum_k |a_ik - muA| |b_kj - muB|, relative to U:
      2 (2^-24 + 2^-52)      fp32 rounding of each centred, scaled operand (after the fp64 subtraction);
      2^-20                  the tf32 split: hi + lo misses a' by <= 2^-22 |a'|, and lo lo' <= 2^-22 |a'||b'| is dropped;
      3 L 2^-23 (1 + 2^-8)   fp32 accumulation of the 3 L products of a chunk of L <= 2048 (truncating, any order);
      (K + chunks + 8) 2^-52 fp64: chunk re-accumulation, line sums and corrections, the final rounding;
    plus K 2^(sA + sB - 120) for the values, products and partial sums below 2^-126 (scaled) that are flushed or lost."""
    A, B = np.asarray(A, dtype=np.float64), np.asarray(B, dtype=np.float64)
    K = A.shape[1]
    L = min(CHUNK, -(-K // 32) * 32)
    chunks = -(-K // CHUNK)
    sA, sB = scale_exp(A), scale_exp(B)
    ld = np.longdouble
    # scaled magnitudes (<= 4), so that U itself cannot overflow; the scale is applied in extended precision
    xa = np.ldexp(np.abs(A) + abs(mu[0]), -sA)
    xb = np.ldexp(np.abs(B) + abs(mu[1]), -sB)
    U = xa @ xb
    rel = 2 * (2.0 ** -24 + 2.0 ** -52) + 2.0 ** -20 + 3 * L * 2.0 ** -23 * (1 + 2.0 ** -8) + (K + chunks + 8) * 2.0 ** -52
    E = (ld(1.01 * rel) * U.astype(ld) + ld(K) * ld(2.0) ** -120) * ld(2.0) ** (sA + sB)
    return np.minimum(E, ld(np.finfo(np.float64).max)).astype(np.float64) + 4 * 2.0 ** -1074


# ---------------------------------------------------------------------------------------------------------------- simulation
def _rz32(x):
    """fp64 array -> nearest fp32 toward zero (as fp64)."""
    r = x.astype(np.float32)
    over = np.abs(r.astype(np.float64)) > np.abs(x)
    r[over] = np.nextafter(r[over], np.float32(0))
    return r.astype(np.float64)


def _add_rz32(acc, p):
    """fl32 toward zero of the exact acc + p (acc fp32 values, p exact products, both fp64 arrays): TwoSum keeps the part of
    the sum that fp64 rounded away, so a result exact in fp64 but not in fp32 is truncated correctly either way."""
    s = acc + p
    bb = s - acc
    err = (acc - (s - bb)) + (p - bb)
    r = _rz32(s)
    back = (r == s) & (err != 0) & (np.sign(err) != np.sign(s)) & (s != 0)
    r[back] = np.nextafter(r[back].astype(np.float32), np.float32(0)).astype(np.float64)
    return r


def simulate_truncating(A, B, mu=(0.0, 0.0)):
    """The device arithmetic with an fp32 accumulator that truncates every addition, in the kernel's order: per chunk the pairs
    lo hi', hi lo', hi hi', each over k ascending, into one accumulator.  O(n m K) numpy work: small sizes only."""
    A, B = np.asarray(A, dtype=np.float64), np.asarray(B, dtype=np.float64)
    n, K = A.shape
    sA, sB = scale_exp(A), scale_exp(B)
    a, ha, la = prepare(A, mu[0], sA)
    b, hb, lb = prepare(B, mu[1], sB)
    rc, cc = _corrections(a, sA, b, sB, mu, K)
    C = None
    for k0 in range(0, K, CHUNK):
        acc = np.zeros((n, B.shape[1]))
        for x, y in ((la, hb), (ha, lb), (ha, hb)):
            for k in range(k0, min(K, k0 + CHUNK)):
                acc = _add_rz32(acc, np.outer(x[:, k].astype(np.float64), y[k].astype(np.float64)))
        term = np.ldexp(acc, sA + sB)
        C = term + (rc[:, None] + cc[None, :]) if C is None else C + term
    return C

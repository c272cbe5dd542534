"""GPU tests of the Ozaki-II fp64 multiply (gemm_algo 0 / 4) on irregular block shapes and extreme values.

Every numeric case is held to three checks (check_product):
  (a) block ids, presence, shapes and flags equal the oracle's;
  (b) the WHOLE product against numpy fp64 within oz2_bound + the classical bound of numpy's own dot products -- an indexing
      error anywhere shows;
  (c) EXACT entries (tests/exact_ref.py) within oz2_bound alone at sampled positions and next to every tile / slot / block
      boundary; integer-valued inputs must give the exact product bit for bit.
The operand width alpha comes from the documented rule (exact_ref.alpha_of / moduli_for), never from the device."""
from fractions import Fraction

import numpy as np
import pytest

import matrel_b200 as mb
from oracle import matrel_oracle as O
from tests.exact_ref import alpha_of, exact_entries, fp64_dot_bound, moduli_for, oz2_bound, round_to_double
from tests.util import REL_TOL, assert_same_dataset, from_dataset, to_dataset

pytestmark = pytest.mark.gpu

DEFAULTS = {"gemm_algo": 4, "crt_moduli": 0, "ozaki_scratch_mb": 0, "gemm_variant": -1, "oz2_ksplit": 0}
TINY = 2.0 ** -1074


@pytest.fixture(scope="module")
def sess():
    s = mb.MatfastSession(device=0, gemm_algo=4)
    yield s
    s.stop()


def multiply(s, A, B, n, k, m, blk, **opts):
    """The product as a block dict plus the statistics of the call; options are restored afterwards."""
    for key, v in {**DEFAULTS, **opts}.items():
        s.set_option(key, v)
    try:
        s.reset_stats()
        got = from_dataset(to_dataset(s, A).matrixMultiply(n, k, to_dataset(s, B), k, m, blk))
        return got, s.stats()
    finally:
        for key, v in DEFAULTS.items():
            s.set_option(key, v)


def random_mask(rng, p):
    table = rng.random((64, 64)) < p
    return lambda i, j: bool(table[i % 64, j % 64])


def to_blocks(M, blk, tmask=lambda i, j: False, absent=()):
    """Block dict of the dense array M: block (i, j) row-major where tmask(i, j), left out where (i, j) is in `absent`."""
    n, m = M.shape
    out = {}
    for i in range(-(-n // blk)):
        for j in range(-(-m // blk)):
            if (i, j) in absent:
                continue
            sub = M[i * blk:(i + 1) * blk, j * blk:(j + 1) * blk]
            if tmask(i, j):
                out[(i, j)] = O.DenseMatrix(sub.shape[0], sub.shape[1], np.ascontiguousarray(sub).reshape(-1), True)
            else:
                out[(i, j)] = O.DenseMatrix(sub.shape[0], sub.shape[1], np.ascontiguousarray(sub.T).reshape(-1), False)
    return out


def without(M, blk, absent):
    M = M.copy()
    for (i, j) in absent:
        M[i * blk:(i + 1) * blk, j * blk:(j + 1) * blk] = 0.0
    return M


def edge_indices(n, blk):
    """Rows / columns next to a 128-row tile, 256-column tile, slot or block boundary, and the last one."""
    idx = {0, n - 1}
    for b0 in range(0, n, blk):
        for local in range(0, min(blk, n - b0) + 1, 128):
            idx.update((b0 + local - 1, b0 + local))
        idx.update((b0 - 1, b0, min(n, b0 + blk) - 1))
    return sorted(i for i in idx if 0 <= i < n)


def positions(rng, n, m, blk, samples=300, cap=500):
    rows, cols = edge_indices(n, blk), edge_indices(m, blk)
    grid = [(i, j) for i in rows for j in cols]
    if len(grid) > cap:
        grid = [grid[t] for t in rng.choice(len(grid), cap, replace=False)]
    pos = set(grid) | {(n - 1, m - 1), (0, 0), (n - 1, 0), (0, m - 1)}
    pos |= {(i, int(rng.integers(m))) for i in rows} | {(int(rng.integers(n)), j) for j in cols}   # every edge row and column
    pos |= {(int(rng.integers(n)), m - 1) for _ in range(8)}
    pos |= {(int(rng.integers(n)), int(rng.integers(m))) for _ in range(samples)}
    return sorted(pos)


def within(got, exact, bound):
    """|got - exact| <= bound with got an fp64 value, exact a Fraction; non-finite values must be the correctly rounded exact one."""
    want = round_to_double(exact)
    if not (np.isfinite(got) and np.isfinite(want)):
        return got == want
    if not np.isfinite(bound):
        return True
    return abs(Fraction(float(got)) - exact) <= Fraction(float(bound))


def check_product(got, Af, Bf, blk, A, B, alpha, rng, *, samples=300, extra=None, integer=False, whole=True):
    """Af, Bf: the operands as dense arrays with absent blocks zeroed; A, B: the block dicts that were multiplied.
    extra: additional allowance (array), e.g. the fp64 bound when the exact kernel may have produced the blocks."""
    n, k = Af.shape
    m = Bf.shape[1]
    want = O.matrix_multiply(A, n, k, B, k, m, blk)
    assert_same_dataset(got, want, tol=REL_TOL)                                   # (a)
    G = O.assemble(got, n, m, blk)
    with np.errstate(over="ignore", invalid="ignore"):
        ref = Af @ Bf
        op = oz2_bound(Af, Bf, alpha, np.zeros((n, m)))
        if extra is not None:
            op = op + extra
        if integer:
            exact = (Af.astype(object) @ Bf.astype(object)).astype(np.float64)
            assert np.array_equal(G, exact)
            return G
        if whole:                                                                 # (b)
            fin = np.isfinite(ref)
            assert np.array_equal(G[~fin], ref[~fin], equal_nan=True)
            bound = op + 2.0 ** -52 * np.abs(ref) + fp64_dot_bound(Af, Bf)
            bad = fin & ~(np.abs(G - ref) <= bound)
            assert not bad.any(), ("whole product", np.argwhere(bad)[:5].tolist(), float(np.max(np.abs(G - ref)[bad] / bound[bad])))
    pos = positions(rng, n, m, blk, samples)                                      # (c)
    with np.errstate(over="ignore"):
        for (i, j), x in zip(pos, exact_entries(Af, Bf, pos)):
            want = round_to_double(x)
            assert within(G[i, j], x, op[i, j] + 2.0 ** -52 * abs(want)), ("exact entry", i, j, float(G[i, j]), want, float(op[i, j]))
    return G


def uniform_pair(rng, n, k, m):
    return rng.uniform(-1, 1, (n, k)), rng.uniform(-1, 1, (k, m))


# ------------------------------------------------------------------------------------------------ shapes
SHAPES = [
    # n, k, m, blk, absent A blocks, absent B blocks
    (563, 563, 563, 200, (), ()),                      # ss 256 (CTA pairs): block smaller than its slot, ragged edges
    (563, 563, 563, 200, ((1, 1), (0, 2)), ((2, 0), (1, 1))),
    (2000, 2000, 2000, 1000, (), ()),                  # ss 1024
    (2001, 2001, 2001, 1000, (), ()),                  # last block row / column of one line: a padding tile
    (356, 300, 356, 256, (), ()),                      # last block row of 100 rows: one tile plus the padding tile
    (488, 300, 488, 256, (), ()),                      # last block row of 232 rows
    (513, 700, 513, 512, (), ()),                      # last block row of 1 row
    (641, 700, 641, 512, (), ()),                      # last block row of 129 rows: two tiles, no padding
    (900, 500, 900, 384, (), ()),                      # ss 384 (single CTA): every other n-tile straddles two column slots
    (800, 450, 800, 300, (), ()),                      # ss 384 with blocks smaller than the slot
    (1, 300, 500, 256, (), ()),                        # M = 1
    (500, 300, 1, 256, (), ()),                        # N = 1
    (300, 1, 260, 256, (), ()),                        # inner dimension of one block: the outer-product path, K = 1 ...
    (300, 31, 260, 256, (), ()),
    (300, 129, 260, 256, (), ()),
    (300, 1000, 260, 1024, (), ()),
]


@pytest.mark.parametrize("n,k,m,blk,absA,absB", SHAPES, ids=["%dx%dx%d-blk%d-%s" % (*c[:4], "sparse" if c[4] else "full") for c in SHAPES])
def test_irregular_shapes_meet_the_bound(sess, n, k, m, blk, absA, absB):
    rng = np.random.default_rng(n * 7 + k * 3 + m + blk + len(absA))
    Af, Bf = uniform_pair(rng, n, k, m)
    A, B = to_blocks(Af, blk, random_mask(rng, 0.5), absA), to_blocks(Bf, blk, random_mask(rng, 0.5), absB)
    Af, Bf = without(Af, blk, absA), without(Bf, blk, absB)
    got, st = multiply(sess, A, B, n, k, m, blk)
    assert st["tc_gemm_launches"] == 1 and st["tc_moduli"] == moduli_for(k)
    check_product(got, Af, Bf, blk, A, B, alpha_of(moduli_for(k), k), rng)


@pytest.mark.parametrize("variant", ["absent_right", "absent_left", "zero_block"])
def test_straddled_tile_with_one_side_missing(sess, variant):
    """ss = 384: the n-tile of columns 256..511 covers the end of column slot 0 and the start of slot 1.  Remove (or zero) the
    blocks of B so that an output block on one side of such a tile does not exist while the other does."""
    rng = np.random.default_rng(len(variant))
    n, k, m, blk = 700, 384, 1100, 384
    Af, Bf = uniform_pair(rng, n, k, m)
    absB = {"absent_right": ((0, 1),), "absent_left": ((0, 0),), "zero_block": ()}[variant]
    if variant == "zero_block":
        Bf[:, 384:768] = 0.0
    A, B = to_blocks(Af, blk, random_mask(rng, 0.5)), to_blocks(Bf, blk, random_mask(rng, 0.5), absB)
    Bf = without(Bf, blk, absB)
    got, st = multiply(sess, A, B, n, k, m, blk)
    assert st["tc_gemm_launches"] == 1
    assert ((0, 1) in got) == (variant != "absent_right") and ((0, 0) in got) == (variant != "absent_left")
    check_product(got, Af, Bf, blk, A, B, alpha_of(14, k), rng)


@pytest.mark.parametrize("n,k,m,blk", [(563, 333, 421, 200), (300, 1000, 513, 512), (800, 450, 641, 300)])
def test_integer_data_is_bit_exact_on_irregular_shapes(sess, n, k, m, blk):
    rng = np.random.default_rng(blk)
    Af = rng.integers(-(1 << 20), 1 << 20, (n, k)).astype(np.float64)
    Bf = rng.integers(-(1 << 20), 1 << 20, (k, m)).astype(np.float64)
    A, B = to_blocks(Af, blk, random_mask(rng, 0.5)), to_blocks(Bf, blk, random_mask(rng, 0.5))
    got, st = multiply(sess, A, B, n, k, m, blk)
    assert st["tc_gemm_launches"] == 1
    check_product(got, Af, Bf, blk, A, B, alpha_of(14, k), rng, integer=True)


@pytest.mark.parametrize("k", [255, 256, 257, 4096, 4097, 65536, 131071])
def test_inner_dimension_sets_moduli_and_alpha(sess, k):
    """The operand width changes with ceil(log2 K): one case on either side of each step, held to the bound of ITS alpha."""
    rng = np.random.default_rng(k)
    n, m, blk = 100, 90, 1024                                       # blocks far smaller than the slot, padding tiles, K % 128 != 0
    Af, Bf = uniform_pair(rng, n, k, m)
    A, B = to_blocks(Af, blk, random_mask(rng, 0.5)), to_blocks(Bf, blk, random_mask(rng, 0.5))
    got, st = multiply(sess, A, B, n, k, m, blk)
    T = moduli_for(k)
    assert st["tc_gemm_launches"] == 1 and st["tc_moduli"] == T
    check_product(got, Af, Bf, blk, A, B, alpha_of(T, k), rng, samples=300 if k <= 4097 else 6)


def test_inner_dimension_beyond_the_accumulator_range_stays_on_the_exact_kernel(sess):
    rng = np.random.default_rng(8)
    n, k, m, blk = 40, 1 << 17, 30, 1024
    Af, Bf = uniform_pair(rng, n, k, m)
    A, B = to_blocks(Af, blk), to_blocks(Bf, blk)
    got, st = multiply(sess, A, B, n, k, m, blk)
    assert st["tc_gemm_launches"] == 0
    assert_same_dataset(got, O.matrix_multiply(A, n, k, B, k, m, blk), tol=1e-11)
    assert np.all(np.abs(O.assemble(got, n, m, blk) - Af @ Bf) <= 2 * fp64_dot_bound(Af, Bf))


# ------------------------------------------------------------------------------------------------ result-neutral options
def same_bits(got, ref):
    assert_same_dataset(got, {k: O.DenseMatrix(v.numRows, v.numCols, v.values) for k, v in ref.items()}, exact_storage=True)


@pytest.mark.parametrize("n,k,m,blk,small_mb", [
    (563, 563, 563, 200, 8),        # K spans 5 chunks of 128 (odd: the K-split order must decline)
    (600, 1000, 700, 256, 12),      # 8 chunks (even)
])
def test_execution_options_do_not_change_a_bit(sess, n, k, m, blk, small_mb):
    rng = np.random.default_rng(n + k)
    Af, Bf = uniform_pair(rng, n, k, m)
    A, B = to_blocks(Af, blk, random_mask(rng, 0.5)), to_blocks(Bf, blk, random_mask(rng, 0.5))
    ref, st = multiply(sess, A, B, n, k, m, blk)
    assert st["tc_gemm_launches"] == 1
    check_product(ref, Af, Bf, blk, A, B, alpha_of(14, k), rng, samples=50)
    for opts in ({"oz2_ksplit": 1}, {"oz2_ksplit": 2}, {"gemm_variant": 2}, {"ozaki_scratch_mb": small_mb}):
        got, st = multiply(sess, A, B, n, k, m, blk, **opts)
        assert st["tc_gemm_launches"] == 1, opts
        same_bits(got, ref)


def test_pipelined_ingest_of_a_ragged_shape_is_bit_identical(sess):
    import torch
    rng = np.random.default_rng(77)
    n, k, m, blk = 963, 963, 963, 200
    Af, Bf = uniform_pair(rng, n, k, m)
    A, B = to_blocks(Af, blk, random_mask(rng, 0.5)), to_blocks(Bf, blk, random_mask(rng, 0.5))
    ref, _ = multiply(sess, A, B, n, k, m, blk)
    check_product(ref, Af, Bf, blk, A, B, alpha_of(14, k), rng, samples=50)
    pin = lambda x: mb.DenseMatrix(x.numRows, x.numCols, torch.from_numpy(x.values).pin_memory().numpy(), x.isTransposed)  # noqa: E731
    pA = [mb.MatrixBlock(i, j, pin(x)) for (i, j), x in A.items()]
    pB = [mb.MatrixBlock(i, j, pin(x)) for (i, j), x in B.items()]
    sess.reset_stats()
    dA, dB = sess.emptyDataset(), sess.emptyDataset()
    for t in range(-(-n // blk)):
        dA.put_blocks([b for b in pA if b.rid == t])
        dB.put_blocks([b for b in pB if b.cid == t])
    got = from_dataset(dA.matrixMultiply(n, k, dB, k, m, blk))
    assert sess.stats()["tc_gemm_launches"] == 1
    same_bits(got, ref)


# ------------------------------------------------------------------------------------------------ values
def v_tiny_rows(rng, n, k, m):
    Af, Bf = uniform_pair(rng, n, k, m)
    return Af * np.exp2(rng.integers(-1010, -900, n))[:, None], Bf * np.exp2(rng.integers(0, 50, m))[None, :]


def v_subnormals(rng, n, k, m):
    Af, Bf = uniform_pair(rng, n, k, m)
    for i in (3, 127, 128, n - 1):                                  # whole rows of sub-normals (29 bits of range at most)
        Af[i, :] = rng.integers(1 << 30, 1 << 40, k) * TINY * rng.choice([-1.0, 1.0], k)
    for j in (0, 255, m - 2):
        Bf[:, j] = rng.integers(1 << 25, 1 << 35, k) * TINY
    Af[10, 7], Af[200, k - 1], Bf[5, 9], Bf[k - 1, 300] = 5 * TINY, -TINY, 3 * TINY, 2.0 ** -1040   # isolated ones
    return Af, Bf


def v_huge_rows(rng, n, k, m):
    Af, Bf = uniform_pair(rng, n, k, m)
    Af[::5, :] *= 2.0 ** 1023
    Af[n - 1, :] *= 2.0 ** 1023
    Af[5, 11] = np.finfo(np.float64).max
    Af[n - 1, k - 1] = -np.finfo(np.float64).max
    return Af, Bf * 2.0 ** -20


def v_overflow(rng, n, k, m):
    """Rows 4 and n-1 of A times columns 6 and m-1 of B exceed the fp64 range (by a factor of hundreds); everything else is finite."""
    Af, Bf = uniform_pair(rng, n, k, m)
    Bf *= 2.0 ** -20
    Af[4, :] = rng.uniform(1, 2, k) * 2.0 ** 1022
    Af[n - 1, :] = -rng.uniform(1, 2, k) * 2.0 ** 1022
    Bf[:, 6] = rng.uniform(1, 2, k)
    Bf[:, m - 1] = -rng.uniform(1, 2, k)
    return Af, Bf


def v_subnormal_results(rng, n, k, m):
    Af, Bf = uniform_pair(rng, n, k, m)
    return Af * np.exp2(rng.integers(-530, -510, n))[:, None], Bf * np.exp2(rng.integers(-530, -510, m))[None, :]


def v_power_of_two_maxima(rng, n, k, m):
    """Line maxima exactly 2^q (scaled integer 2^(alpha-1)) or the fp64 value just below (which rounds UP to 2^alpha, the largest
    scaled magnitude the CRT range allows); one row / column made of nothing but that value."""
    Af, Bf = rng.uniform(-0.5, 0.5, (n, k)), rng.uniform(-0.5, 0.5, (k, m))
    for i in range(n):
        q = float(2.0 ** rng.integers(-8, 8))
        Af[i] *= q
        Af[i, rng.integers(k)] = q if i % 2 else np.nextafter(q, 0.0)
    for j in range(m):
        q = float(2.0 ** rng.integers(-8, 8))
        Bf[:, j] *= q
        Bf[rng.integers(k), j] = -q if j % 2 else -np.nextafter(q, 0.0)
    Af[7, :] = np.nextafter(8.0, 0.0)
    Bf[:, 9] = np.nextafter(0.25, 0.0)
    Af[n - 1, :] = -4.0
    Bf[:, m - 1] = 2.0
    return Af, Bf


def v_zeros(rng, n, k, m):
    Af, Bf = uniform_pair(rng, n, k, m)
    Af[rng.random((n, k)) < 0.05] = -0.0
    Bf[rng.random((k, m)) < 0.05] = -0.0
    Af[[0, 129, 199, 200, n - 1], :] = 0.0                           # all-zero rows / columns inside non-zero blocks
    Bf[:, [1, 255, 256, m - 1]] = 0.0
    Af[:, 17] = 0.0
    Bf[300, :] = -0.0
    Af[50, :], Af[50, k - 1] = 0.0, 3.5                              # lines with a single non-zero
    Bf[:, 70], Bf[0, 70] = 0.0, -1.25e-3
    return Af, Bf


def v_cancellation(rng, n, k, m):
    """Triples (a, -a/2, -a/2) against (b, b, b) sum to zero exactly -- while their roundings to alpha bits do not cancel -- so the
    product is carried by one or two terms of 2^-20 b although |A||B| is of order K."""
    Af, Bf = rng.uniform(1, 2, (n, k)), rng.uniform(1, 2, (k, m))
    g = (k - 1) // 3
    Af[:, 1:3 * g:3] = Af[:, 2:3 * g:3] = -0.5 * Af[:, 0:3 * g:3]
    Bf[1:3 * g:3, :] = Bf[2:3 * g:3, :] = Bf[0:3 * g:3, :]
    Af[:, 3 * g:] = 2.0 ** -20
    return Af, Bf


VALUE_CASES = {"tiny_rows": v_tiny_rows, "subnormals": v_subnormals, "huge_rows": v_huge_rows, "overflow": v_overflow,
               "subnormal_results": v_subnormal_results, "power_of_two_maxima": v_power_of_two_maxima, "zeros": v_zeros,
               "cancellation": v_cancellation}
# unguarded at a small paired ragged shape; auto-selected (range guard on) at a size above the 2^33-flop threshold
VALUE_SHAPES = {4: (563, 563, 563, 200), 0: (1700, 1700, 1700, 200)}


@pytest.mark.parametrize("algo", [4, 0])
@pytest.mark.parametrize("case", sorted(VALUE_CASES))
def test_extreme_values_meet_the_bound(sess, case, algo):
    n, k, m, blk = VALUE_SHAPES[algo]
    rng = np.random.default_rng(len(case) * 31 + algo)
    Af, Bf = VALUE_CASES[case](rng, n, k, m)
    A, B = to_blocks(Af, blk, random_mask(rng, 0.5)), to_blocks(Bf, blk, random_mask(rng, 0.5))
    got, st = multiply(sess, A, B, n, k, m, blk, gemm_algo=algo)
    assert st["tc_gemm_launches"] == 1 and st["tc_moduli"] == moduli_for(k)
    # under the guard the isolated sub-normals are multiplied in fp64 and added to the result: a few more roundings of |A||B|
    with np.errstate(over="ignore"):
        extra = 2.0 ** -50 * (np.abs(Af) @ np.abs(Bf)) if algo == 0 and case == "subnormals" else None
    G = check_product(got, Af, Bf, blk, A, B, alpha_of(14, k), rng, extra=extra)
    if case == "overflow":
        assert G[4, 6] == np.inf and G[4, m - 1] == -np.inf and G[n - 1, 6] == -np.inf and G[n - 1, m - 1] == np.inf
        assert np.isinf(G).sum() == 4


@pytest.mark.parametrize("algo", [4, 0])
def test_nonfinite_operands_follow_ieee(sess, algo):
    n, k, m, blk = VALUE_SHAPES[algo]
    rng = np.random.default_rng(algo)
    Af, Bf = uniform_pair(rng, n, k, m)
    Af[3, 5], Af[n - 1, k - 1] = np.inf, np.nan                      # the second one inside the ragged corner block
    Bf[k - 1, m - 1], Bf[7, 300], Bf[200, 0] = -np.inf, np.nan, np.inf
    A, B = to_blocks(Af, blk, random_mask(rng, 0.5)), to_blocks(Bf, blk, random_mask(rng, 0.5))
    got, _ = multiply(sess, A, B, n, k, m, blk, gemm_algo=algo)
    assert_same_dataset(got, O.matrix_multiply(A, n, k, B, k, m, blk), tol=1e-11)
    G = O.assemble(got, n, m, blk)
    with np.errstate(invalid="ignore"):
        ref = Af @ Bf
    assert np.array_equal(np.isnan(G), np.isnan(ref)) and np.array_equal(G[np.isinf(ref)], ref[np.isinf(ref)])


# ------------------------------------------------------------------------------------------------ range guard and fix-up
GN, GBLK = 1700, 200                                              # 2 * 1700^3 flops: above the auto threshold; last block 100 wide
G_ALPHA = alpha_of(14, GN)
RANGE_BITS = G_ALPHA - 18
CHECKER = lambda i, j: (i + j) % 2 == 0                          # noqa: E731  row-major blocks where i + j is even


def guard_operands(rng):
    """Rows of A with maximum exactly 1 (so depths below the maximum are plain exponents); B in [1, 2)."""
    Af, Bf = rng.uniform(0.25, 1.0, (GN, GN)), rng.uniform(1.0, 2.0, (GN, GN))
    Af[:, 0] = 1.0
    return Af, Bf


def lone_column(Bf, j, ks, rng):
    """Column j of B zero except at rows ks: C(i, j) consists of the products a(i, ks) b(ks, j) only."""
    Bf[:, j] = 0.0
    Bf[ks, j] = rng.uniform(1.0, 2.0, len(ks))


def guard_run(sess, Af, Bf, algo=0):
    A, B = to_blocks(Af, GBLK, CHECKER), to_blocks(Bf, GBLK, CHECKER)
    got, st = multiply(sess, A, B, GN, GN, GN, GBLK, gemm_algo=algo)
    assert st["tc_gemm_launches"] == 1
    return got, A, B


def test_range_threshold_one_binade_inside_and_one_outside(sess):
    rng = np.random.default_rng(1)
    Af, Bf = guard_operands(rng)
    mant = 1.0 + rng.integers(1, 1 << 52, 2) * 2.0 ** -52              # full 53-bit significands
    Af[10, 400] = mant[0] * 2.0 ** -RANGE_BITS                          # range_bits binades below the row maximum: kept in the residues
    Af[11, 400] = mant[1] * 2.0 ** -(RANGE_BITS + 1)                    # one more: multiplied exactly
    lone_column(Bf, 33, [400], rng)
    got, A, B = guard_run(sess, Af, Bf)
    G = check_product(got, Af, Bf, GBLK, A, B, G_ALPHA, rng, samples=100)
    inside, outside = exact_entries(Af, Bf, [(10, 33), (11, 33)])
    assert G[11, 33] == round_to_double(outside)
    err = abs(Fraction(float(G[10, 33])) - inside)
    assert 0 < err <= Fraction(2) ** -G_ALPHA * Fraction(float(Bf[400, 33]) * 1.01)    # rounded to a multiple of 2^(1 - alpha): row maximum 1


def outlier_operands(rng, count):
    """`count` elements of block row 0 of A, 2^-45 below their row maximum, each facing a lone element of B."""
    Af, Bf = guard_operands(rng)
    spots = [(int(i), 300 + 3 * t, 40 + t) for t, i in enumerate(rng.integers(0, GBLK, count))]   # (row, k, column)
    for (i, k, j) in spots:
        Af[i, k] = rng.uniform(1.0, 2.0) * 2.0 ** -45
        lone_column(Bf, j, [k], rng)
    return Af, Bf, spots


def test_a_full_record_table_keeps_the_tensor_core_result(sess):
    rng = np.random.default_rng(64)
    Af, Bf, spots = outlier_operands(rng, 64)
    got, A, B = guard_run(sess, Af, Bf)
    G = check_product(got, Af, Bf, GBLK, A, B, G_ALPHA, rng, samples=100)
    absAB = np.abs(Af) @ np.abs(Bf)
    for (i, _, j), x in zip(spots, exact_entries(Af, Bf, [(i, j) for i, _, j in spots])):
        assert within(G[i, j], x, 2.0 ** -50 * absAB[i, j]), (i, j)
    unguarded = O.assemble(guard_run(sess, Af, Bf, algo=4)[0], GN, GN, GBLK)
    touched = np.zeros((GN, GN), dtype=bool)
    touched[[i for i, _, _ in spots], :] = True
    assert np.array_equal(G[~touched], unguarded[~touched])          # the tensor-core result was kept
    assert max(abs(unguarded[i, j] - G[i, j]) / abs(G[i, j]) for i, _, j in spots) > 1e-3   # ... which alone loses those products


def test_one_record_too_many_falls_back_to_the_exact_kernel(sess):
    rng = np.random.default_rng(65)
    Af, Bf, spots = outlier_operands(rng, 65)
    got, A, B = guard_run(sess, Af, Bf)
    want = O.matrix_multiply(A, GN, GN, B, GN, GN, GBLK)
    assert_same_dataset(got, want, tol=1e-11)
    G = O.assemble(got, GN, GN, GBLK)
    assert np.all(np.abs(G - Af @ Bf) <= 2 * fp64_dot_bound(Af, Bf))
    bound = fp64_dot_bound(Af, Bf)
    pos = [(i, j) for i, _, j in spots] + positions(rng, GN, GN, GBLK, samples=50, cap=100)
    for (i, j), x in zip(pos, exact_entries(Af, Bf, pos)):
        assert within(G[i, j], x, bound[i, j]), (i, j)


def test_outliers_in_row_major_and_ragged_edge_blocks(sess):
    rng = np.random.default_rng(3)
    Af, Bf = guard_operands(rng)
    last = GN - 1
    tiny = lambda: rng.uniform(1.0, 2.0) * 2.0 ** -45               # noqa: E731
    # (i, k) of A: row-major block (0, 2); column-major block (0, 3); the ragged corner block (8, 8), row-major; last row, column-major
    a_spots = [(5, 450), (6, 700), (last, last), (last - 1, 1500)]
    for (i, k) in a_spots:
        assert CHECKER(i // GBLK, k // GBLK) == ((i, k) in (a_spots[0], a_spots[2]))
        Af[i, k] = tiny()
    for t, (i, k) in enumerate(a_spots):
        lone_column(Bf, 60 + 400 * t, [k], rng)                      # columns 60, 460, 860, 1260
    # outliers of B: Bf has entries in [1, 2), so 2^-45 times that is far below every column maximum
    b_spots = [(450, 900), (last, last), (700, 1300), (123, last - 3)]   # (k, j): same k as an outlier of A; ragged corner; ...
    for (k, j) in b_spots:
        Bf[k, j] = tiny()
    # an outlier of B facing an outlier of A, and nothing else in that dot product: the pair must be counted exactly once
    lone_column(Bf, 1660, [450, 20], rng)
    Bf[450, 1660] *= 2.0 ** -45
    Af[5, 20] = 0.0
    got, A, B = guard_run(sess, Af, Bf)
    G = check_product(got, Af, Bf, GBLK, A, B, G_ALPHA, rng, samples=100)
    absAB = np.abs(Af) @ np.abs(Bf)
    pos = [(5, 60), (6, 460), (last, 860), (last - 1, 1260), (5, 1660)]   # entries made of one exact outlier product each
    for (i, j), x in zip(pos, exact_entries(Af, Bf, pos)):
        assert within(G[i, j], x, 2.0 ** -50 * absAB[i, j]), (i, j)
    unguarded = O.assemble(guard_run(sess, Af, Bf, algo=4)[0], GN, GN, GBLK)
    touched = np.zeros((GN, GN), dtype=bool)
    touched[[i for i, _ in a_spots], :] = True
    touched[:, [j for _, j in b_spots] + [1660]] = True
    assert np.array_equal(G[~touched], unguarded[~touched])

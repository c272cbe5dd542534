"""GPU tests of the Ozaki-I fp64 multiply (gemm_algo 2, ozaki_slices 2 .. 7) on irregular shapes, slice counts and extreme values.

Every case on the Ozaki-I path is held to three checks (check_product), and its route is asserted from the launch counters
(5 + S kernel launches: two absmax passes, the exponents, two slice passes, one GEMM per diagonal):
  (a) block ids, presence, shapes and flags equal the oracle's, and so do the positions of non-finite values;
  (b) the WHOLE product equals tests/ozaki1_ref.ozaki1_model bit for bit, signed zeros included -- the model replays the device
      arithmetic on the operand blocks the kernel sees (seen_operands);
  (c) EXACT entries (tests/exact_ref.py) next to every 128-row tile, 256-column tile and block edge, plus random samples, are
      within ozaki1_bound.
Cases that must leave the path (Inf / NaN, K S >= 2^17, a sparse x dense partial) are bit-identical to gemm_algo 1."""
import numpy as np
import pytest

import matrel_b200 as mb
from oracle import matrel_oracle as O
from tests.exact_ref import exact_entries, round_to_double
from tests.ozaki1_ref import clamp_slices, ozaki1_bound, ozaki1_model, seen_operands
from tests.test_gpu_ozaki2_edges import positions, random_mask, to_blocks, within
from tests.test_gpu_streamed import _streamed
from tests.test_gpu_unaligned import adopt_unaligned
from tests.util import REL_TOL, assert_same_dataset, from_dataset, to_dataset

pytestmark = pytest.mark.gpu

TINY = 2.0 ** -1074
DEFAULTS = {"gemm_algo": 2, "ozaki_slices": 7}


@pytest.fixture(scope="module")
def sess():
    s = mb.MatfastSession(device=0, gemm_algo=2)
    yield s
    s.stop()


def run(s, dA, dB, n, k, m, blk, **opts):
    """dA x dB (datasets) as a block dict plus the statistics of the call; options are restored afterwards."""
    for key, v in {**DEFAULTS, **opts}.items():
        s.set_option(key, v)
    try:
        s.reset_stats()
        got = from_dataset(dA.matrixMultiply(n, k, dB, k, m, blk))
        return got, s.stats()
    finally:
        for key, v in DEFAULTS.items():
            s.set_option(key, v)


def multiply(s, A, B, n, k, m, blk, **opts):
    return run(s, to_dataset(s, A), to_dataset(s, B), n, k, m, blk, **opts)


def assert_ozaki1_route(st, S, densify=0):
    assert st["gemm_launches"] == 1 and st["tc_gemm_launches"] == 0, st
    assert st["kernel_launches"] == 5 + S + densify, (st["kernel_launches"], 5 + S + densify)


def bits(x):
    return np.ascontiguousarray(x, dtype=np.float64).view(np.int64)


def check_product(got, A, B, n, k, m, blk, S, rng, *, samples=100, cap=200, oracle=True):
    """(a), (b), (c) of the module docstring; returns the assembled product.  All three are evaluated before any is asserted, so
    that a failure reports the size of the error against the bound as well as the bit mismatch."""
    S = clamp_slices(S)
    oracle_error = None
    if oracle:                                                                    # (a); the values are (b)'s and (c)'s
        try:
            assert_same_dataset(got, O.matrix_multiply(A, n, k, B, k, m, blk), tol=np.inf)
        except AssertionError as e:
            oracle_error = str(e)[:300]
    Af, Bf = seen_operands(A, B, n, k, m, blk)
    G = O.assemble(got, n, m, blk)
    model = ozaki1_model(Af, Bf, S)
    mismatch = bits(G) != bits(model)                                             # (b)
    pos = positions(rng, n, m, blk, samples, cap)                                 # (c)
    bound = ozaki1_bound(Af, Bf, S, np.zeros((n, m)))
    worst, outside = 0.0, []
    with np.errstate(over="ignore"):
        for (i, j), x in zip(pos, exact_entries(Af, Bf, pos)):
            lim = bound[i, j] + 2.0 ** -52 * abs(round_to_double(x))
            if not within(G[i, j], x, lim):
                outside.append((i, j, float(G[i, j]), round_to_double(x)))
            if np.isfinite(G[i, j]) and np.isfinite(lim) and lim > 0:
                worst = max(worst, abs(float(G[i, j]) - round_to_double(x)) / lim)
    report = {"oracle": oracle_error, "bits_differ": int(mismatch.sum()), "first": np.argwhere(mismatch)[:3].tolist(), "outside_bound": len(outside),
              "first_outside": outside[:3], "worst_error_over_bound": worst}
    assert oracle_error is None and not mismatch.any() and not outside, report
    return G


def uniform_pair(rng, n, k, m):
    return rng.uniform(-1, 1, (n, k)), rng.uniform(-1, 1, (k, m))


# ------------------------------------------------------------------------------------------------ shapes
SHAPES = [
    # n, k, m, blk, S, absent A blocks, absent B blocks
    (130, 120, 140, 50, 7, (), ()),                    # blk not a multiple of 4: byte-wise digit stores; tiles straddle blocks
    (300, 200, 260, 64, 5, (), ()),
    (400, 270, 390, 130, 7, (), ()),                   # blk = 2 mod 4
    (563, 563, 563, 200, 6, ((1, 1), (0, 2)), ((2, 0), (1, 1))),
    (700, 520, 600, 256, 3, (), ()),
    (1100, 1050, 700, 1001, 4, (), ()),                # one ragged block of 99 / 49 behind a 1001 block
    (1, 300, 500, 64, 7, (), ()),                      # M = 1
    (500, 300, 1, 64, 7, (), ()),                      # N = 1
    (300, 1, 260, 256, 7, (), ()),                     # K = 1: one block column, the outer-product path
    (300, 31, 260, 256, 2, (), ()),                    # outer product, K % 4 != 0
    (300, 129, 260, 100, 7, (), ()),                   # K one past a 128-byte stage, ragged
]


@pytest.mark.parametrize("n,k,m,blk,S,absA,absB", SHAPES, ids=["%dx%dx%d-blk%d-S%d-%s" % (*c[:5], "sparse" if c[5] else "full") for c in SHAPES])
def test_irregular_shapes(sess, n, k, m, blk, S, absA, absB):
    rng = np.random.default_rng(n * 7 + k * 3 + m + blk + S)
    Af, Bf = uniform_pair(rng, n, k, m)
    A, B = to_blocks(Af, blk, random_mask(rng, 0.5), absA), to_blocks(Bf, blk, random_mask(rng, 0.5), absB)
    got, st = multiply(sess, A, B, n, k, m, blk, ozaki_slices=S)
    assert_ozaki1_route(st, S)
    check_product(got, A, B, n, k, m, blk, S, rng)


@pytest.mark.parametrize("layout", ["column_major", "row_major"])
def test_one_layout_throughout(sess, layout):
    rng = np.random.default_rng(len(layout))
    n, k, m, blk = 450, 333, 517, 150
    Af, Bf = uniform_pair(rng, n, k, m)
    tm = (lambda i, j: layout == "row_major")
    A, B = to_blocks(Af, blk, tm), to_blocks(Bf, blk, tm)
    got, st = multiply(sess, A, B, n, k, m, blk)
    assert_ozaki1_route(st, 7)
    check_product(got, A, B, n, k, m, blk, 7, rng)


def test_absent_block_rows_and_columns_and_zero_blocks(sess):
    """Block row 1 of A and block column 2 of B are absent (the compacted slots skip them); two blocks are all zero."""
    rng = np.random.default_rng(11)
    n, k, m, blk = 640, 400, 700, 128
    Af, Bf = uniform_pair(rng, n, k, m)
    absA = tuple((1, j) for j in range(4))
    absB = tuple((i, 2) for i in range(4))
    Af[3 * blk:4 * blk, 0:blk] = 0.0
    Bf[blk:2 * blk, 4 * blk:5 * blk] = -0.0
    A, B = to_blocks(Af, blk, random_mask(rng, 0.5), absA), to_blocks(Bf, blk, random_mask(rng, 0.5), absB)
    got, st = multiply(sess, A, B, n, k, m, blk)
    assert_ozaki1_route(st, 7)
    assert not any(key[0] == 1 or key[1] == 2 for key in got)
    check_product(got, A, B, n, k, m, blk, 7, rng)


def test_a_block_that_meets_nothing_sets_no_exponent(sess):
    """A block of A holding 2^900 whose block row of B is absent is no operand of the kernel: its rows are bit for bit those of the
    product without that block."""
    rng = np.random.default_rng(12)
    n, k, m, blk = 400, 500, 300, 128
    Af, Bf = uniform_pair(rng, n, k, m)
    Af[130, 2 * blk + 7] = 2.0 ** 900
    A, B = to_blocks(Af, blk, random_mask(rng, 0.5)), to_blocks(Bf, blk, random_mask(rng, 0.5), tuple((2, j) for j in range(3)))
    got, st = multiply(sess, A, B, n, k, m, blk)
    assert_ozaki1_route(st, 7)
    check_product(got, A, B, n, k, m, blk, 7, rng)
    A2 = {key: x for key, x in A.items() if key[1] != 2}
    ref, _ = multiply(sess, A2, B, n, k, m, blk)
    for key in ref:
        assert np.array_equal(bits(got[key].values), bits(ref[key].values)), key


def test_more_than_65535_blocks_per_operand(sess):
    """256 x 16400 and 16400 x 256 in blocks of 8: 65,600 blocks each, so the absmax and slice passes run in two grid chunks."""
    rng = np.random.default_rng(13)
    n, k, m, blk, S = 256, 16400, 256, 8, 2
    Af, Bf = uniform_pair(rng, n, k, m)
    A, B = to_blocks(Af, blk, random_mask(rng, 0.5)), to_blocks(Bf, blk, random_mask(rng, 0.5))
    assert len(A) > 65535 and len(B) > 65535
    got, st = multiply(sess, A, B, n, k, m, blk, ozaki_slices=S)
    assert_ozaki1_route(st, S)
    # (a) without the oracle's 2 million block products: every output block, dense, column-major, full size
    assert sorted(got) == [(i, j) for i in range(n // blk) for j in range(m // blk)]
    assert all(isinstance(x, mb.DenseMatrix) and not x.isTransposed and (x.numRows, x.numCols) == (blk, blk) for x in got.values())
    check_product(got, A, B, n, k, m, blk, S, rng, samples=10, cap=10, oracle=False)


@pytest.mark.parametrize("n,k,m,blk", [(200, 168, 136, 64), (199, 131, 93, 67)])
def test_unaligned_adopted_blocks(sess, n, k, m, blk):
    rng = np.random.default_rng(n)
    Af, Bf = rng.uniform(-1, 1, (n, k)), rng.uniform(-1, 1, (k, m))
    A, B = to_blocks(Af, blk, random_mask(rng, 0.5)), to_blocks(Bf, blk, random_mask(rng, 0.5))
    dA, ka = adopt_unaligned(sess, A)
    dB, kb = adopt_unaligned(sess, B)
    got, st = run(sess, dA, dB, n, k, m, blk)
    del dA, dB, ka, kb
    assert_ozaki1_route(st, 7)
    check_product(got, A, B, n, k, m, blk, 7, rng)


# ------------------------------------------------------------------------------------------------ slices
SL_SHAPE = (330, 290, 310, 100)


@pytest.mark.parametrize("S", [2, 3, 4, 5, 6, 7])
def test_every_slice_count(sess, S):
    n, k, m, blk = SL_SHAPE
    rng = np.random.default_rng(40 + S)
    Af, Bf = uniform_pair(rng, n, k, m)
    Af *= np.exp2(rng.integers(-20, 20, n))[:, None]
    A, B = to_blocks(Af, blk, random_mask(rng, 0.5)), to_blocks(Bf, blk, random_mask(rng, 0.5))
    got, st = multiply(sess, A, B, n, k, m, blk, ozaki_slices=S)
    assert_ozaki1_route(st, S)
    check_product(got, A, B, n, k, m, blk, S, rng)


@pytest.mark.parametrize("asked,means", [(1, 2), (9, 7), (0, 7)])
def test_slice_count_clamps(sess, asked, means):
    n, k, m, blk = SL_SHAPE
    rng = np.random.default_rng(50 + asked)
    Af, Bf = uniform_pair(rng, n, k, m)
    A, B = to_blocks(Af, blk, random_mask(rng, 0.5)), to_blocks(Bf, blk, random_mask(rng, 0.5))
    got, st = multiply(sess, A, B, n, k, m, blk, ozaki_slices=asked)
    assert_ozaki1_route(st, means)
    ref, _ = multiply(sess, A, B, n, k, m, blk, ozaki_slices=means)
    for key in ref:
        assert np.array_equal(bits(got[key].values), bits(ref[key].values)), key
    check_product(got, A, B, n, k, m, blk, means, rng, samples=30)


def saturating_pair(S, n, K, m, rng):
    """Lines whose S - 1 low digits are all -128 and whose top digit is +-64 (tests/test_ozaki1_ref_cpu.py), alternating signs in
    one row: every accumulator term is as large as an s32 term can be."""
    X = float(64 * 256 ** (S - 1) - 128 * (256 ** (S - 1) - 1) // 255)
    Af = np.ldexp(X, rng.integers(-30, 30, n) + 2 - 8 * S)[:, None] * np.ones((n, K))
    Bf = -np.ldexp(X, rng.integers(-30, 30, m) + 2 - 8 * S)[None, :] * np.ones((K, m))
    Af[1] *= np.where(np.arange(K) % 2 == 0, 1.0, -1.0)
    return Af, Bf


@pytest.mark.parametrize("S", [2, 7])
def test_accumulator_limit(sess, S):
    """K S < 2^17 at the largest K stays on Ozaki-I, bit-exact to the model; one more K leaves for the exact DMMA kernel."""
    rng = np.random.default_rng(60 + S)
    n, m, blk = 24, 20, 4096
    K = ((1 << 17) - 1) // S
    Af, Bf = saturating_pair(S, n, K + 1, m, rng)
    A, B = to_blocks(Af[:, :K], blk), to_blocks(Bf[:K], blk)
    got, st = multiply(sess, A, B, n, K, m, blk, ozaki_slices=S)
    assert_ozaki1_route(st, S)
    check_product(got, A, B, n, K, m, blk, S, rng, samples=8, cap=8)
    A, B = to_blocks(Af, blk), to_blocks(Bf, blk)
    got, st = multiply(sess, A, B, n, K + 1, m, blk, ozaki_slices=S)
    dmma, st1 = multiply(sess, A, B, n, K + 1, m, blk, gemm_algo=1)
    assert st["kernel_launches"] == st1["kernel_launches"]                       # declined before any Ozaki-I launch
    for key in dmma:
        assert np.array_equal(bits(got[key].values), bits(dmma[key].values)), key


# ------------------------------------------------------------------------------------------------ values
def v_range300(rng, n, k, m):
    Af, Bf = uniform_pair(rng, n, k, m)
    return Af * np.exp2(rng.integers(-300, 300, (n, k))), Bf * np.exp2(rng.integers(-300, 300, (k, m)))


def v_huge_rows(rng, n, k, m):
    """Rows with maximum >= 2^1023 (one of exactly 1.5 2^1023, one at the largest finite value) times columns of ~2^-1000."""
    Af, Bf = uniform_pair(rng, n, k, m)
    Af[::7] *= 2.0 ** 1023
    Af[3, 5] = 1.5 * 2.0 ** 1023
    Af[n - 1, k - 1] = -np.finfo(np.float64).max
    return Af, Bf * 2.0 ** -1000


def v_huge_columns(rng, n, k, m):
    Bt, At = v_huge_rows(rng, m, k, n)
    return At.T.copy(), Bt.T.copy()


def v_tiny_rows(rng, n, k, m):
    """Rows of tiny normal values (2^-1016 .. 2^-1060) and rows of sub-normals times columns near 2^1000."""
    Af, Bf = uniform_pair(rng, n, k, m)
    Af = Af * np.exp2(rng.integers(-1060, -1016, n).astype(float))[:, None]
    Af[::5] = rng.integers(-(1 << 30), 1 << 30, (len(Af[::5]), k)) * TINY
    Af[1, :] = 2.0 ** -1016 * rng.uniform(1, 2, k)
    return Af, Bf * 2.0 ** 1000 * rng.uniform(1, 1.9, m)[None, :]


def v_tiny_columns(rng, n, k, m):
    Bt, At = v_tiny_rows(rng, m, k, n)
    return At.T.copy(), Bt.T.copy()


def v_subnormal_results(rng, n, k, m):
    Af, Bf = uniform_pair(rng, n, k, m)
    return Af * np.exp2(rng.integers(-530, -510, n))[:, None], Bf * np.exp2(rng.integers(-530, -510, m))[None, :]


def v_cancellation(rng, n, k, m):
    """Triples (a, -a/2, -a/2) against (b, b, b) cancel exactly; the product is carried by 2^-20 terms."""
    Af, Bf = rng.uniform(1, 2, (n, k)), rng.uniform(1, 2, (k, m))
    g = (k - 1) // 3
    Af[:, 1:3 * g:3] = Af[:, 2:3 * g:3] = -0.5 * Af[:, 0:3 * g:3]
    Bf[1:3 * g:3, :] = Bf[2:3 * g:3, :] = Bf[0:3 * g:3, :]
    Af[:, 3 * g:] = 2.0 ** -20
    return Af, Bf


def v_zeros(rng, n, k, m):
    Af, Bf = uniform_pair(rng, n, k, m)
    Af[rng.random((n, k)) < 0.05] = -0.0
    Bf[rng.random((k, m)) < 0.05] = -0.0
    Af[[0, 127, 128, n - 1], :] = -0.0                               # all-zero rows and columns, of negative zeros
    Bf[:, [1, 255, 256, m - 1]] = 0.0
    Af[50, :], Af[50, k - 1] = -0.0, -3.5                            # lines with a single non-zero
    Bf[:, 70], Bf[0, 70] = -0.0, 1.25e-3
    return Af, Bf


def v_near_max(rng, n, k, m):
    """Pairs (row i_t of A, column j_t of B) whose only large entries a_t over [1, 2) 2^511 and b_t = 0.995 DBL_MAX / a_t meet at
    k_t, everything else ~2^400: C(i_t, j_t) is 0.995 of the largest double, and for about a third of them the top-digit term alone
    exceeds the fp64 range."""
    Af, Bf = rng.uniform(-1, 1, (n, k)) * 2.0 ** 400, rng.uniform(-1, 1, (k, m)) * 2.0 ** 400
    T = min(n, k, m) - 10
    i, kk, j = rng.permutation(n)[:T], rng.permutation(k)[:T], rng.permutation(m)[:T]
    a = rng.uniform(1, 2, T) * 2.0 ** 511
    Af[i, kk], Bf[kk, j] = a, 0.995 * np.finfo(np.float64).max / a
    return Af, Bf


VALUE_CASES = {"near_max": v_near_max, "range300": v_range300, "huge_rows": v_huge_rows, "huge_columns": v_huge_columns, "tiny_rows": v_tiny_rows,
               "tiny_columns": v_tiny_columns, "subnormal_results": v_subnormal_results, "cancellation": v_cancellation,
               "zeros": v_zeros}
V_SHAPE = (330, 290, 310, 100)


@pytest.mark.parametrize("S", [3, 7])
@pytest.mark.parametrize("case", sorted(VALUE_CASES))
def test_extreme_values(sess, case, S):
    n, k, m, blk = V_SHAPE
    rng = np.random.default_rng(len(case) * 31 + S)
    Af, Bf = VALUE_CASES[case](rng, n, k, m)
    assert np.isfinite(Af).all() and np.isfinite(Bf).all()
    A, B = to_blocks(Af, blk, random_mask(rng, 0.5)), to_blocks(Bf, blk, random_mask(rng, 0.5))
    got, st = multiply(sess, A, B, n, k, m, blk, ozaki_slices=S)
    assert_ozaki1_route(st, S)
    G = check_product(got, A, B, n, k, m, blk, S, rng)
    assert np.isfinite(G).all()
    if case == "zeros":                                             # an all-zero accumulator gives +0, whatever the operands' zeros
        for i in (0, 127, 128, n - 1):
            assert not np.signbit(G[i]).any()
        for j in (1, 255, 256, m - 1):
            assert not np.signbit(G[:, j]).any()


@pytest.mark.parametrize("side", ["A", "B"])
def test_nonfinite_operands_fall_back_to_the_exact_kernel(sess, side):
    n, k, m, blk = V_SHAPE
    rng = np.random.default_rng(len(side))
    Af, Bf = uniform_pair(rng, n, k, m)
    if side == "A":
        Af[3, 5], Af[n - 1, k - 1] = np.inf, np.nan
    else:
        Bf[k - 1, m - 1], Bf[7, 200] = -np.inf, np.nan
    A, B = to_blocks(Af, blk, random_mask(rng, 0.5)), to_blocks(Bf, blk, random_mask(rng, 0.5))
    got, st = multiply(sess, A, B, n, k, m, blk)
    dmma, st1 = multiply(sess, A, B, n, k, m, blk, gemm_algo=1)
    assert st["kernel_launches"] == st1["kernel_launches"] + 3             # absmax x 2 + exponents, then the exact kernel
    for key in dmma:
        assert np.array_equal(bits(got[key].values), bits(dmma[key].values)), key


# ------------------------------------------------------------------------------------------------ routes and paths
def sparse_of(x, csr=False):
    """CSC (or CSR) block of the oracle DenseMatrix x."""
    a = x.to_numpy()
    if csr:
        return O.DenseMatrix(a.shape[1], a.shape[0], np.ascontiguousarray(a).reshape(-1)).toSparse().transpose()
    return O.DenseMatrix(a.shape[0], a.shape[1], np.ascontiguousarray(a.T).reshape(-1)).toSparse()


def test_a_sparse_times_dense_partial_keeps_the_product_on_the_exact_kernel(sess):
    rng = np.random.default_rng(70)
    n, k, m, blk = 400, 300, 350, 128
    Af, Bf = uniform_pair(rng, n, k, m)
    Af[rng.random((n, k)) < 0.97] = 0.0
    A, B = to_blocks(Af, blk), to_blocks(Bf, blk)
    A[(1, 1)] = sparse_of(A[(1, 1)], csr=True)                    # CSR: the sparse x dense kernel adds without atomics
    got, st = multiply(sess, A, B, n, k, m, blk)
    dmma, st1 = multiply(sess, A, B, n, k, m, blk, gemm_algo=1)
    for key in ("kernel_launches", "gemm_launches", "tc_gemm_launches"):      # no Ozaki-I launch: the route of gemm_algo 1
        assert st[key] == st1[key], (key, st[key], st1[key])
    assert sorted(got) == sorted(dmma)
    for key in dmma:
        assert np.array_equal(bits(got[key].values), bits(dmma[key].values)), key


def test_densified_sparse_operands_take_ozaki1(sess):
    """Sparse x sparse above the 0.1 density threshold, and dense x sparse above the dense x sparse route's density: both are
    GEMM pairs of the dense images.  The sparse blocks of A sit in block column 0, whose block row of B is all sparse, so that no
    sparse x dense pair sends the product to the exact kernel."""
    rng = np.random.default_rng(71)
    n, k, m, blk = 400, 300, 350, 128
    Af, Bf = uniform_pair(rng, n, k, m)
    Af[rng.random((n, k)) < 0.5] = 0.0
    Bf[rng.random((k, m)) < 0.7] = 0.0
    A, B = to_blocks(Af, blk), to_blocks(Bf, blk)
    for key in ((0, 0), (2, 0)):
        A[key] = sparse_of(A[key], csr=key[0] == 2)
    for key in ((0, 0), (0, 1), (0, 2), (1, 1), (2, 2)):
        B[key] = sparse_of(B[key], csr=key == (1, 1))
    got, st = multiply(sess, A, B, n, k, m, blk)
    assert_ozaki1_route(st, 7, densify=7)                         # one dense-image launch per sparse block
    check_product(got, A, B, n, k, m, blk, 7, rng)


def test_multiply_right_after_pipelined_ingest_is_bit_identical(sess):
    import torch
    rng = np.random.default_rng(77)
    n, k, m, blk = 963, 700, 800, 200
    Af, Bf = uniform_pair(rng, n, k, m)
    A, B = to_blocks(Af, blk, random_mask(rng, 0.5)), to_blocks(Bf, blk, random_mask(rng, 0.5))
    ref, st = multiply(sess, A, B, n, k, m, blk)
    assert_ozaki1_route(st, 7)
    check_product(ref, A, B, n, k, m, blk, 7, rng, samples=30)
    pin = lambda x: mb.DenseMatrix(x.numRows, x.numCols, torch.from_numpy(x.values).pin_memory().numpy(), x.isTransposed)  # noqa: E731
    pA = [mb.MatrixBlock(i, j, pin(x)) for (i, j), x in A.items()]
    pB = [mb.MatrixBlock(i, j, pin(x)) for (i, j), x in B.items()]
    dA, dB = sess.emptyDataset(), sess.emptyDataset()
    for t in range(-(-max(n, m) // blk)):
        dA.put_blocks([b for b in pA if b.rid == t])
        dB.put_blocks([b for b in pB if b.cid == t])
    got, st = run(sess, dA, dB, n, k, m, blk)
    assert_ozaki1_route(st, 7)
    for key in ref:
        assert np.array_equal(bits(got[key].values), bits(ref[key].values)), key


def test_streamed_product_is_within_the_bound():
    """Host-resident operands, C tile by tile: each tile takes its own line exponents (never larger than the whole product's), so
    the bound of the whole product holds at the exact entries."""
    rng = np.random.default_rng(78)
    n, k, m, blk = 900, 600, 800, 200
    Af, Bf = uniform_pair(rng, n, k, m)
    Af *= np.exp2(rng.integers(-30, 30, n))[:, None]
    A, B = to_blocks(Af, blk, random_mask(rng, 0.5)), to_blocks(Bf, blk, random_mask(rng, 0.5))
    with mb.MatfastSession(device=0, gemm_algo=2) as s:
        host = lambda ds: s.createHostDataset([mb.MatrixBlock(i, j, mb.DenseMatrix(v.numRows, v.numCols, v.values, v.isTransposed))  # noqa: E731
                                               for (i, j), v in sorted(ds.items())])
        C, st = _streamed(s, host(A), host(B), n, k, m, blk)
        assert C.isHost and st["stream_tiles"] >= 2 and st["tc_gemm_launches"] == 0
        assert st["kernel_launches"] >= st["stream_tiles"] * (5 + 7)            # every tile on Ozaki-I
        got = from_dataset(C)
    assert_same_dataset(got, O.matrix_multiply(A, n, k, B, k, m, blk), tol=REL_TOL)
    Af, Bf = seen_operands(A, B, n, k, m, blk)
    G = O.assemble(got, n, m, blk)
    bound = ozaki1_bound(Af, Bf, 7, np.zeros((n, m)))
    pos = positions(rng, n, m, blk, 100, 200)
    for (i, j), x in zip(pos, exact_entries(Af, Bf, pos)):
        assert within(G[i, j], x, bound[i, j] + 2.0 ** -52 * abs(round_to_double(x))), (i, j)

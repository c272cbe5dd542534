"""GPU tests of the Gram route (DESIGN section 4.1.2): C = A^T A and C = A A^T over the arrays A.t() shares with A.

The reference is the general route on a copy (A.multiplyScalar(1.0): the same bits in other arrays, so the route is not taken).
Every case asserts:
  - every block of C bit for bit equal to the reference (NaN positions only where non-finite), with the same ids, shapes and flags;
  - C == C^T bit for bit on the assembled matrix;
  - the route: gram_blocks, gram_mirrored_blocks, tc_int8_ops against the tile rule of tests/gram_ref.py, and the launch count;
  - a second run giving the same bits.
Look-alikes must leave both counters at zero."""
from fractions import Fraction

import numpy as np
import pytest

import matrel_b200 as mb
from tests.exact_ref import exact_entries, moduli_for
from tests.gram_ref import gram_int8_ops
from tests.util import from_dataset, to_dataset
from oracle import matrel_oracle as O

pytestmark = pytest.mark.gpu

DEFAULTS = {"gemm_algo": 0, "crt_moduli": 0, "ozaki_scratch_mb": 0, "gemm_variant": -1, "oz2_ksplit": 0}


@pytest.fixture(scope="module")
def sess():
    s = mb.MatfastSession(device=0)
    yield s
    s.stop()


def to_blocks(M, blk, tmask=lambda i, j: False, absent=()):
    out = {}
    for i in range(-(-M.shape[0] // blk)):
        for j in range(-(-M.shape[1] // blk)):
            if (i, j) in absent:
                continue
            sub = M[i * blk:(i + 1) * blk, j * blk:(j + 1) * blk]
            vals = np.ascontiguousarray(sub if tmask(i, j) else sub.T).reshape(-1)
            out[(i, j)] = O.DenseMatrix(sub.shape[0], sub.shape[1], vals, bool(tmask(i, j)))
    return out


def run(s, L, R, dims, blk, **opts):
    for k, v in {**DEFAULTS, **opts}.items():
        s.set_option(k, v)
    try:
        s.reset_stats()
        C = L.matrixMultiply(dims[0], dims[1], R, dims[2], dims[3], blk)
        s.sync()
        return C, s.stats()
    finally:
        for k, v in DEFAULTS.items():
            s.set_option(k, v)


def bits(x):
    x = np.asarray(x, dtype=np.float64)
    return np.where(np.isnan(x), np.nan, x).view(np.int64)   # NaN payloads are not compared


def assert_same_bits(got, ref):
    g, r = from_dataset(got), from_dataset(ref)
    assert sorted(g) == sorted(r)
    for key, w in r.items():
        v = g[key]
        assert (v.numRows, v.numCols, v.isTransposed) == (w.numRows, w.numCols, w.isTransposed) == (w.numRows, w.numCols, False), key
        assert isinstance(v, mb.DenseMatrix), key
        assert np.array_equal(bits(v.values), bits(w.values)), key
    return g


def assert_symmetric(C, N, blk):
    G = C.toNumpy(N, N, blk)
    assert np.array_equal(bits(G), bits(G.T))
    return G


def gram_and_ref(s, Af, blk, kind, tmask=lambda i, j: False, absent=()):
    """(left, right, dims) of the Gram product and of its reference on a copy."""
    A = to_dataset(s, to_blocks(Af, blk, tmask, absent))
    A2 = A.multiplyScalar(1.0)
    m, n = Af.shape
    if kind == "AtA":
        return (A.t(), A, (n, m, m, n)), (A2.t(), A, (n, m, m, n)), n
    return (A, A.t(), (m, n, n, m)), (A, A2.t(), (m, n, n, m)), m


def expected_counts(C):
    ids = list(from_dataset(C))
    return sum(i <= j for i, j in ids), sum(i > j for i, j in ids)


def check_gram(s, Af, blk, kind, *, tmask=lambda i, j: False, absent=(), expect_oz2, **opts):
    """Runs the case; returns the assembled C.  Launches: the mirror pass adds one; on Ozaki-II the shared residues save the
    three A-side preparation launches (absmax, exponents, residues) of a resident product."""
    (L, R, dims), (L2, R2, _), N = gram_and_ref(s, Af, blk, kind, tmask, absent)
    ref, st_ref = run(s, L2, R2, dims, blk, **opts)
    got, st = run(s, L, R, dims, blk, **opts)
    g = assert_same_bits(got, ref)
    G = assert_symmetric(got, N, blk)
    up, low = expected_counts(got)
    assert (st["gram_blocks"], st["gram_mirrored_blocks"]) == (up, low)
    assert (st_ref["gram_blocks"], st_ref["gram_mirrored_blocks"]) == (0, 0)
    assert st["tc_gemm_launches"] == st_ref["tc_gemm_launches"] == (1 if expect_oz2 else 0)
    if expect_oz2:
        K = dims[1]
        order = sorted({i for i, _ in g})
        slot = {b: t for t, b in enumerate(order)}
        dimsl = [g[(b, b)].numRows for b in order]
        outs = [(slot[i], slot[j]) for i, j in g]
        assert st["tc_int8_ops"] == gram_int8_ops(dimsl, outs, blk, moduli_for(K), K)
        assert st["kernel_launches"] == st_ref["kernel_launches"] + 1 - 3
    else:
        assert st["kernel_launches"] == st_ref["kernel_launches"] + 1
    again, _ = run(s, L, R, dims, blk, **opts)
    assert_same_bits(again, got)
    return G


def uniform(rng, m, n):
    return rng.uniform(-1.0, 1.0, (m, n))


@pytest.mark.parametrize("kind,m,n,blk,algo,oz2", [
    ("AtA", 2048, 2048, 1024, 4, True),     # paired CTA tiles, whole blocks
    ("AAt", 3000, 1500, 512, 4, True),      # tall A, ragged last block row
    ("AtA", 1500, 2000, 640, 4, True),      # slot stride 640: tiles straddle slots, single-CTA kernel
    ("AtA", 700, 2500, 1024, 4, True),      # one k-block: the outer product
    ("AAt", 2600, 2100, 512, 0, True),      # auto above 2^33 flop: Ozaki-II with the range guard
    ("AtA", 1000, 1000, 256, 0, False),     # auto below 2^33 flop: DMMA
    ("AAt", 1500, 1100, 512, 1, False),     # DMMA by request
    ("AtA", 900, 1300, 640, 1, False),
])
def test_gram_is_the_general_product_bit_for_bit(sess, kind, m, n, blk, algo, oz2):
    rng = np.random.default_rng(m + n + blk)
    check_gram(sess, uniform(rng, m, n), blk, kind, expect_oz2=oz2, gemm_algo=algo)


@pytest.mark.parametrize("algo,oz2", [(4, True), (1, False)])
def test_absent_blocks_and_mixed_layouts(sess, algo, oz2):
    rng = np.random.default_rng(5)
    table = rng.random((8, 8)) < 0.5
    check_gram(sess, uniform(rng, 1800, 1900), 512, "AtA", tmask=lambda i, j: bool(table[i, j]),
               absent={(0, 1), (2, 3), (3, 0)}, expect_oz2=oz2, gemm_algo=algo)


def oz2_bytes(blk, K, T, nslots, tiles, share):
    ss = -(-blk // 128) * 128
    kpad = -(-K // 128) * 128
    npad = -(-(ss * nslots) // 256) * 256
    return T * ((0 if share else ss * nslots) + npad) * kpad + T * tiles * 128 * 256


def test_scratch_that_panels_the_general_route_keeps_the_gram_route_resident(sess):
    rng = np.random.default_rng(11)
    blk, m, n = 512, 2048, 2048
    Af = uniform(rng, m, n)
    T = moduli_for(m)
    tiles = (4 * 512 // 128) * (4 * 512 // 256)
    mb_budget = -(-(oz2_bytes(blk, m, T, 4, tiles, True) + oz2_bytes(blk, m, T, 4, tiles, False)) // 2 // (1 << 20))
    assert oz2_bytes(blk, m, T, 4, tiles, True) <= mb_budget << 20 < oz2_bytes(blk, m, T, 4, tiles, False)
    (L, R, dims), (L2, R2, _), N = gram_and_ref(sess, Af, blk, "AtA")
    ref_small, st_ref_small = run(sess, L2, R2, dims, blk, gemm_algo=4, ozaki_scratch_mb=mb_budget)
    _, st_ref_full = run(sess, L2, R2, dims, blk, gemm_algo=4)
    got_small, st_small = run(sess, L, R, dims, blk, gemm_algo=4, ozaki_scratch_mb=mb_budget)
    _, st_full = run(sess, L, R, dims, blk, gemm_algo=4)
    assert st_ref_small["kernel_launches"] > st_ref_full["kernel_launches"]   # the general route panels ...
    assert st_small["kernel_launches"] == st_full["kernel_launches"]          # ... the Gram route stays resident
    assert st_small["gram_blocks"] == 10 and st_small["gram_mirrored_blocks"] == 6
    assert_same_bits(got_small, ref_small)
    assert_symmetric(got_small, N, blk)


def test_range_guard_outliers_on_both_lines(sess):
    """Columns of A with an element 2^-45 below the column maximum: C(p, q) gets exact outlier terms from its row line when column
    p has one and from its column line when column q has one.  Where both do, the general route's order of those terms differs
    between C(p, q) and C(q, p); the Gram route is symmetric there and held to the exact product.  Elsewhere: bit for bit."""
    rng = np.random.default_rng(21)
    m, n, blk = 1700, 1700, 512
    Af = rng.uniform(0.25, 1.0, (m, n))
    Af[0, :] = 1.0
    cols = [3, 40, 700, 1650]
    for t, c in enumerate(cols):
        Af[100 + 7 * t, c] = rng.uniform(1.0, 2.0) * 2.0 ** -45
    (L, R, dims), (L2, R2, _), N = gram_and_ref(sess, Af, blk, "AtA")
    ref, _ = run(sess, L2, R2, dims, blk, gemm_algo=0)
    got, st = run(sess, L, R, dims, blk, gemm_algo=0)
    assert st["tc_gemm_launches"] == 1 and st["gram_blocks"] == 10
    G = assert_symmetric(got, N, blk)
    Gr = ref.toNumpy(N, N, blk)
    both = np.zeros((N, N), dtype=bool)
    both[np.ix_(cols, cols)] = True
    assert np.array_equal(bits(G[~both]), bits(Gr[~both]))
    assert np.array_equal(bits(np.triu(G)), bits(np.triu(Gr)))         # on and above the diagonal: the general route's own bits
    pos = [(p, q) for p in cols for q in cols]
    absAB = np.abs(Af.T) @ np.abs(Af)
    for (p, q), x in zip(pos, exact_entries(Af.T, Af, pos)):
        assert abs(Fraction(float(G[p, q])) - x) <= Fraction(float(2.0 ** -50 * absAB[p, q])), (p, q)


def test_nonfinite_operands_fall_back_with_the_route(sess):
    rng = np.random.default_rng(31)
    Af = uniform(rng, 2100, 2100)
    Af[5, 7], Af[1500, 1000], Af[900, 1999] = np.nan, np.inf, -np.inf
    G = check_gram(sess, Af, 512, "AAt", expect_oz2=True, gemm_algo=0)
    assert np.isnan(G).any()


def test_pipelined_multiply_of_operands_still_arriving(sess):
    import torch
    rng = np.random.default_rng(41)
    m, n, blk = 2500, 2300, 512
    Af = uniform(rng, m, n)
    blocks = to_blocks(Af, blk, lambda i, j: (i + j) % 3 == 0)
    pin = lambda x: mb.DenseMatrix(x.numRows, x.numCols, torch.from_numpy(x.values).pin_memory().numpy(), x.isTransposed)  # noqa: E731
    pb = [mb.MatrixBlock(i, j, pin(x)) for (i, j), x in blocks.items()]
    A_ref = to_dataset(sess, blocks)
    for algo in (4, 1):
        sess.set_option("gemm_algo", algo)
        try:
            ref = A_ref.multiplyScalar(1.0).t().matrixMultiply(n, m, A_ref, m, n, blk)
            sess.reset_stats()
            dA = sess.emptyDataset()
            for t in range(-(-m // blk)):
                dA.put_blocks([b for b in pb if b.rid == t])
            got = dA.t().matrixMultiply(n, m, dA, m, n, blk)
            st = sess.stats()
        finally:
            sess.set_option("gemm_algo", 0)
        assert st["gram_blocks"] == 15 and st["gram_mirrored_blocks"] == 10, algo
        assert_same_bits(got, ref)
        assert_symmetric(got, n, blk)


def test_look_alikes_keep_the_general_route(sess):
    rng = np.random.default_rng(51)
    m, n, blk = 1200, 1100, 512
    Af = uniform(rng, m, n)
    A = to_dataset(sess, to_blocks(Af, blk))
    dims = (n, m, m, n)

    def counters(L, R, d=dims, **opts):
        _, st = run(sess, L, R, d, blk, **opts)
        return st["gram_blocks"], st["gram_mirrored_blocks"]

    assert counters(A.t(), A) != (0, 0)                                   # the route itself
    assert counters(A.t(), A.multiplyScalar(1.0)) == (0, 0)              # a copy
    assert counters(A.t(), A.filter_blocks(2, 0)) == (0, 0)               # a subset of the blocks, same arrays
    L = A.t()
    b11 = to_blocks(Af, blk)[(1, 1)]
    L.put_block(1, 1, mb.DenseMatrix(b11.numCols, b11.numRows, b11.values.copy(), True))
    assert counters(L, A) == (0, 0)                                       # one block replaced by a copy
    sp = dict(to_blocks(Af, blk))
    dense = sp[(0, 1)]
    Ab = dense.values.reshape(dense.numCols, dense.numRows).T.copy()
    Ab[np.abs(Ab) < 0.99] = 0.0
    sp[(0, 1)] = O.DenseMatrix(Ab.shape[0], Ab.shape[1], np.ascontiguousarray(Ab.T).reshape(-1)).toSparse()
    S = to_dataset(sess, sp)
    assert counters(S.t(), S) == (0, 0)                                   # a sparse block
    X = to_dataset(sess, to_blocks(uniform(rng, m, 8), blk))
    assert counters(X.t(), X, (8, m, m, 8)) == (0, 0)                    # a thin side: the matrix x vector route
    for algo in (2, 3):
        assert counters(A.t(), A, gemm_algo=algo) == (0, 0)
    assert counters(A.t(), A.toHost()) == (0, 0)                          # a host-resident operand: the streamed multiply

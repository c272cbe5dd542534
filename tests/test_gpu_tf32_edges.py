"""GPU tests of the fp32 multiply (gemm_algo 3, 3xTF32 on wgmma) on irregular shapes, block patterns, extreme values and fallbacks.

Every case on the fp32 path asserts its route from the launch counters (4 + c + ceil(K / 2048) kernel launches: one stats pass
over both operands and its reduction, two slice passes, the correction kernel when the operands are centred (c = 1), one GEMM per K chunk) and
its block ids, presence, shapes and flags against the oracle.  Its values are then held to one of two references
(tests/tf32_ref.py), on the operands the kernel sees (blocks that meet nothing are left out; the means are taken over the
compacted extent, and only when the blocks cover it):
  - operands in the exact regime: the WHOLE product equals tf32_exact_model bit for bit;
  - all other data: every entry is within tf32_bound of the fp64 product (plus that product's own rounding bound), and exact
    entries next to every tile and block edge are within tf32_bound of the exact value.
The bound assumes the tensor core's fp32 accumulator is off by at most 2^-23 of the running magnitude per addition (DESIGN
section 4.3); these cases are the check of that assumption.  Inputs with Inf / NaN, and products with a sparse partial, take the
exact DMMA kernel and are bit-identical to gemm_algo 1."""
import math

import numpy as np
import pytest

import matrel_b200 as mb
from oracle import matrel_oracle as O
from tests.exact_ref import exact_entries, fp64_dot_bound
from tests.test_gpu_ozaki1_edges import bits, sparse_of
from tests.test_gpu_ozaki2_edges import positions, random_mask, to_blocks, within
from tests.test_gpu_streamed import _streamed
from tests.tf32_ref import mean, regime_ok, regime_operand, tf32_bound, tf32_exact_model
from tests.util import assert_same_dataset, from_dataset, rel_err, to_dataset

pytestmark = pytest.mark.gpu
DEFAULTS = {"gemm_algo": 3}


@pytest.fixture(scope="module")
def sess():
    s = mb.MatfastSession(device=0, gemm_algo=3)
    yield s
    s.stop()


def run(s, dA, dB, n, k, m, blk, **opts):
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


def kernel_view(A, B, n, k, m, blk):
    """(Af, Bf, mu, centred): the dense operands the kernel multiplies (blocks that meet no block of the other side left out),
    and the means it uses -- over the compacted extent (block rows of C x K, K x block columns of C), and only when the blocks
    cover that extent."""
    outer = -(-k // blk) == 1
    krows, kcols = {kk for (kk, _) in B}, {kk for (_, kk) in A}
    used_a = {key: x for key, x in A.items() if outer or key[1] in krows}
    used_b = {key: x for key, x in B.items() if outer or key[0] in kcols}
    rows, cols = {i for (i, _) in used_a}, {j for (_, j) in used_b}
    Mc, Nc = sum(min(blk, n - i * blk) for i in rows), sum(min(blk, m - j * blk) for j in cols)
    area = lambda d: sum(x.numRows * x.numCols for x in d.values())  # noqa: E731
    centred = area(used_a) == Mc * k and area(used_b) == k * Nc
    Af, Bf = O.assemble(used_a, n, k, blk), O.assemble(used_b, k, m, blk)
    mu = (mean(Af, Mc * k), mean(Bf, k * Nc)) if centred else (0.0, 0.0)
    return Af, Bf, mu, centred


def assert_tf32_route(st, k, centred, densify=0):
    assert st["gemm_launches"] == 1 and st["tc_gemm_launches"] == 0, st
    want = 4 + int(centred) + -(-k // 2048) + densify
    assert st["kernel_launches"] == want, (st["kernel_launches"], want)


def present(got, n, m, blk):
    mask = np.zeros((n, m), dtype=bool)
    for (i, j) in got:
        mask[i * blk:(i + 1) * blk, j * blk:(j + 1) * blk] = True
    return mask


def check(s, A, B, n, k, m, blk, rng, *, regime=False, oracle=True, samples=100, cap=200, **opts):
    """Multiply on the fp32 path, assert the route, the oracle's structure and the values (module docstring).  Returns the
    assembled product and the worst error over the bound."""
    got, st = multiply(s, A, B, n, k, m, blk, **opts)
    Af, Bf, mu, centred = kernel_view(A, B, n, k, m, blk)
    assert_tf32_route(st, k, centred)
    if oracle:
        assert_same_dataset(got, O.matrix_multiply(A, n, k, B, k, m, blk), tol=np.inf)
    G = O.assemble(got, n, m, blk)
    mask = present(got, n, m, blk)
    if regime:
        assert regime_ok(Af, Bf, mu)
        model = tf32_exact_model(Af, Bf, mu)
        differ = (bits(G) != bits(model)) & mask
        assert not differ.any(), {"bits_differ": int(differ.sum()), "first": np.argwhere(differ)[:3].tolist()}
        return G, 0.0
    E = tf32_bound(Af, Bf, mu)
    with np.errstate(over="ignore", invalid="ignore"):
        ref = Af @ Bf
        lim = E + fp64_dot_bound(Af, Bf)
        err = np.abs(G - ref)
        outside = (~(err <= lim)) & mask
    assert not outside.any(), {"outside": int(outside.sum()), "first": np.argwhere(outside)[:3].tolist()}
    worst = float(np.max(np.where(mask, err / lim, 0.0)))
    pos = [p for p in positions(rng, n, m, blk, samples, cap) if mask[p]]
    for (i, j), x in zip(pos, exact_entries(Af, Bf, pos)):
        assert within(G[i, j], x, E[i, j]), (i, j, float(G[i, j]), float(x), E[i, j])
    return G, worst


def uniform_pair(rng, n, k, m):
    return rng.uniform(-1, 1, (n, k)), rng.uniform(-1, 1, (k, m))


# ------------------------------------------------------------------------------------------------ block sizes and ragged shapes
SHAPES = [  # n, k, m, blk
    (300, 200, 260, 50),
    (254, 300, 258, 127), (256, 300, 256, 128), (258, 300, 260, 129),                  # around the 128-row tile
    (510, 257, 512, 255), (512, 256, 513, 256), (514, 255, 520, 257),                  # around the 256-column tile
    (1300, 700, 1280, 640), (1000, 1100, 900, 1000), (1100, 1024, 1030, 1024),
    (1, 300, 500, 64), (500, 300, 1, 64),                                              # M = 1, N = 1
    (300, 1, 260, 256), (300, 31, 260, 256), (300, 32, 260, 256), (300, 33, 260, 256),   # outer products around Kpad
    (200, 2047, 190, 1000), (200, 2048, 190, 1000), (200, 2049, 190, 1000), (130, 4097, 140, 1000),   # K chunk edges
]


@pytest.mark.parametrize("n,k,m,blk", SHAPES, ids=["%dx%dx%d-blk%d" % c for c in SHAPES])
def test_shapes_within_the_bound(sess, n, k, m, blk):
    rng = np.random.default_rng(n + 3 * k + 7 * m + blk)
    Af, Bf = uniform_pair(rng, n, k, m)
    check(sess, to_blocks(Af, blk, random_mask(rng, 0.5)), to_blocks(Bf, blk, random_mask(rng, 0.5)), n, k, m, blk, rng)


# ------------------------------------------------------------------------------------------------ exact regime, bit for bit
REGIME = [  # n, k, m, blk, offset, exp, absent A blocks, absent B blocks, zero blocks of A
    (256, 512, 128, 100, 0.5, 0, (), (), ()),                       # ragged blocks, centred on an exact mean of 0.5
    (64, 4096, 128, 1000, 0.5, 5, (), (), ()),                      # two K chunks, scaled by 2^5 / 2^-5
    (256, 32, 256, 100, 0.5, -30, (), (), ()),                      # outer product
    (600, 2049, 190, 300, ((1, 2),), (), ((0, 0),)),                # an absent interior block: no centring; a zero block
    (128, 256, 256, 128, 0.5, 0, (), (), ()),                       # one output tile
    (4096, 512, 4096, 512, 0.5, 0, (), (), ()),                     # 512 tiles: many more than SMs
]
REGIME = [c if len(c) == 9 else (*c[:4], 0.0, 0, *c[4:]) for c in REGIME]


@pytest.mark.parametrize("n,k,m,blk,offset,exp,absA,absB,zeroA", REGIME, ids=["%dx%dx%d-blk%d-off%g-exp%d" % c[:6] for c in REGIME])
def test_exact_regime_is_bit_exact(sess, n, k, m, blk, offset, exp, absA, absB, zeroA):
    rng = np.random.default_rng(n + k + m + blk)
    Af = regime_operand(rng, (n, k), density=0.4, offset=offset, exp=exp)
    Bf = regime_operand(rng, (k, m), density=0.4, offset=offset, exp=-exp)
    for (i, j) in zeroA:
        Af[i * blk:(i + 1) * blk, j * blk:(j + 1) * blk] = 0.0
    A, B = to_blocks(Af, blk, random_mask(rng, 0.5), absA), to_blocks(Bf, blk, random_mask(rng, 0.5), absB)
    centred = kernel_view(A, B, n, k, m, blk)[3]
    assert centred == (offset != 0.0)                              # the cases exercise both sides of the centring rule
    check(sess, A, B, n, k, m, blk, rng, regime=True)


def test_absent_block_rows_and_columns_are_compacted(sess):
    """Block row 1 of A and block column 2 of B are absent: the compacted operands are still fully covered, so they are centred
    over the compacted extent; two blocks are all zero."""
    rng = np.random.default_rng(11)
    n, k, m, blk = 640, 400, 700, 128
    Af, Bf = uniform_pair(rng, n, k, m)
    Af, Bf = Af + 0.75, Bf - 0.25
    Af[3 * blk:4 * blk, 0:blk] = 0.0
    Bf[blk:2 * blk, 4 * blk:5 * blk] = -0.0
    A = to_blocks(Af, blk, random_mask(rng, 0.5), tuple((1, j) for j in range(4)))
    B = to_blocks(Bf, blk, random_mask(rng, 0.5), tuple((i, 2) for i in range(4)))
    assert kernel_view(A, B, n, k, m, blk)[3]
    check(sess, A, B, n, k, m, blk, rng)


def test_more_than_65535_blocks_per_operand(sess):
    """256 x 16384 and 16384 x 256 in blocks of 8: 65,536 blocks each, so the stats pass (both operands) runs in three grid chunks and each slice pass in two; the
    regime data make the whole product bit-exact."""
    rng = np.random.default_rng(13)
    n, k, m, blk = 256, 16384, 256, 8
    Af = regime_operand(rng, (n, k), density=0.25, offset=0.5)
    Bf = regime_operand(rng, (k, m), density=0.25, offset=0.5)
    A, B = to_blocks(Af, blk, random_mask(rng, 0.5)), to_blocks(Bf, blk, random_mask(rng, 0.5))
    assert len(A) > 65535 and len(B) > 65535
    G, _ = check(sess, A, B, n, k, m, blk, rng, regime=True, oracle=False)
    assert G.shape == (n, m) and np.count_nonzero(G) > 0.9 * G.size


# ------------------------------------------------------------------------------------------------ values
def test_uniform_long_k_meets_the_tight_bar(sess):
    """U(-1, 1) and 1e6 + U(0, 1) at K = 16384: within 1e-5 of max |C| (BASELINE configs[3]) as well as the bound."""
    n, k, m, blk = 256, 16384, 256, 1024
    for offset in (0.0, 1e6):
        rng = np.random.default_rng(20 + int(offset > 0))
        Af, Bf = uniform_pair(rng, n, k, m)
        if offset:
            Af, Bf = offset + 0.5 * (Af + 1), offset + 0.5 * (Bf + 1)
        G, _ = check(sess, to_blocks(Af, blk, random_mask(rng, 0.5)), to_blocks(Bf, blk, random_mask(rng, 0.5)), n, k, m, blk, rng,
                     samples=20, cap=20)
        assert rel_err(G, Af @ Bf) <= 1e-5, (offset, rel_err(G, Af @ Bf))


def v_cancelling(rng, n, k, m):
    """Rows (a, -a) against columns (b, b), and a 2^-30 tail: C is near 0, carried by the small terms."""
    Af, Bf = rng.uniform(1, 2, (n, k)), rng.uniform(1, 2, (k, m))
    h = k // 2 - 8
    Af[:, h:2 * h] = -Af[:, :h]
    Bf[h:2 * h] = Bf[:h]
    Af[:, 2 * h:] *= 2.0 ** -30
    return Af, Bf


def scaled(ea, eb):
    return lambda rng, n, k, m: (ea * rng.uniform(-1, 1, (n, k)), eb * rng.uniform(-1, 1, (k, m)))


def v_near_max(rng, n, k, m):
    """Operands near 2^511 and 2^505: products up to 2^1016, sum_k |a_ik| |b_kj| near 2^1022, a quarter of the largest double."""
    return rng.uniform(-1, 1, (n, k)) * 2.0 ** 511, rng.uniform(-1, 1, (k, m)) * 2.0 ** 505


VALUES = {"cancelling": v_cancelling, "1e-20": scaled(1e-20, 1e-20), "1e20": scaled(1e20, 1e20), "1e-300x1e300": scaled(1e-300, 1e300),
          "1e300x1e-300": scaled(1e300, 1e-300), "near_max": v_near_max}


@pytest.mark.parametrize("case", sorted(VALUES))
def test_extreme_values_within_the_bound(sess, case):
    n, k, m, blk = 330, 290, 310, 100
    rng = np.random.default_rng(len(case) * 31)
    Af, Bf = VALUES[case](rng, n, k, m)
    G, _ = check(sess, to_blocks(Af, blk, random_mask(rng, 0.5)), to_blocks(Bf, blk, random_mask(rng, 0.5)), n, k, m, blk, rng)
    assert np.isfinite(G).all()
    ref = Af @ Bf
    if case != "cancelling":                                       # the fp32 relative accuracy carries over to every magnitude
        assert rel_err(G, ref) <= 1e-5, rel_err(G, ref)


# ------------------------------------------------------------------------------------------------ fallbacks
@pytest.mark.parametrize("side", ["A", "B"])
@pytest.mark.parametrize("value", [np.inf, np.nan])
def test_nonfinite_operands_fall_back_to_the_exact_kernel(sess, side, value):
    n, k, m, blk = 330, 290, 310, 100
    rng = np.random.default_rng(len(side))
    Af, Bf = uniform_pair(rng, n, k, m)
    if side == "A":
        Af[3, 5] = value
    else:
        Bf[k - 1, m - 1] = -value
    A, B = to_blocks(Af, blk, random_mask(rng, 0.5)), to_blocks(Bf, blk, random_mask(rng, 0.5))
    got, st = multiply(sess, A, B, n, k, m, blk)
    dmma, st1 = multiply(sess, A, B, n, k, m, blk, gemm_algo=1)
    assert st["kernel_launches"] == st1["kernel_launches"] + 2             # stats + their reduction, then the exact kernel
    assert sorted(got) == sorted(dmma)
    for key in dmma:
        assert np.array_equal(bits(got[key].values), bits(dmma[key].values)), key
    G = O.assemble(got, n, m, blk)
    assert np.isfinite(G).sum() > 0.9 * G.size                             # only the affected row / column is non-finite


def test_a_sparse_partial_keeps_the_product_on_the_exact_kernel(sess):
    rng = np.random.default_rng(70)
    n, k, m, blk = 400, 300, 350, 128
    Af, Bf = uniform_pair(rng, n, k, m)
    Af[rng.random((n, k)) < 0.97] = 0.0
    A, B = to_blocks(Af, blk), to_blocks(Bf, blk)
    A[(1, 1)] = sparse_of(A[(1, 1)], csr=True)
    got, st = multiply(sess, A, B, n, k, m, blk)
    dmma, st1 = multiply(sess, A, B, n, k, m, blk, gemm_algo=1)
    for key in ("kernel_launches", "gemm_launches", "tc_gemm_launches"):
        assert st[key] == st1[key], (key, st[key], st1[key])
    for key in dmma:
        assert np.array_equal(bits(got[key].values), bits(dmma[key].values)), key


# ------------------------------------------------------------------------------------------------ run to run, other routes
def test_repeated_call_is_bit_identical(sess):
    """Positive data (the means matter) with 64 blocks along every line: the operand totals and line sums are added in a fixed
    order, so two calls agree to the bit."""
    rng = np.random.default_rng(80)
    n, k, m, blk = 512, 4096, 512, 64
    Af, Bf = rng.uniform(0, 1, (n, k)), rng.uniform(0, 1, (k, m))
    A, B = to_blocks(Af, blk, random_mask(rng, 0.5)), to_blocks(Bf, blk, random_mask(rng, 0.5))
    dA, dB = to_dataset(sess, A), to_dataset(sess, B)
    first, st = run(sess, dA, dB, n, k, m, blk)
    assert_tf32_route(st, k, True)
    for _ in range(2):
        again, _ = run(sess, dA, dB, n, k, m, blk)
        for key in first:
            assert np.array_equal(bits(again[key].values), bits(first[key].values)), key
    Gf = O.assemble(first, n, m, blk)
    assert rel_err(Gf, Af @ Bf) <= 1e-5


def test_multiply_right_after_pipelined_ingest_is_bit_identical(sess):
    import torch
    rng = np.random.default_rng(77)
    n, k, m, blk = 963, 700, 800, 200
    Af, Bf = uniform_pair(rng, n, k, m)
    A, B = to_blocks(Af, blk, random_mask(rng, 0.5)), to_blocks(Bf, blk, random_mask(rng, 0.5))
    ref, _ = multiply(sess, A, B, n, k, m, blk)
    pin = lambda x: mb.DenseMatrix(x.numRows, x.numCols, torch.from_numpy(x.values).pin_memory().numpy(), x.isTransposed)  # noqa: E731
    pA = [mb.MatrixBlock(i, j, pin(x)) for (i, j), x in A.items()]
    pB = [mb.MatrixBlock(i, j, pin(x)) for (i, j), x in B.items()]
    dA, dB = sess.emptyDataset(), sess.emptyDataset()
    for t in range(-(-max(n, m) // blk)):
        dA.put_blocks([b for b in pA if b.rid == t])
        dB.put_blocks([b for b in pB if b.cid == t])
    got, st = run(sess, dA, dB, n, k, m, blk)
    assert_tf32_route(st, k, True)
    for key in ref:
        assert np.array_equal(bits(got[key].values), bits(ref[key].values)), key


def test_streamed_product_is_within_the_bound():
    """Host-resident operands, C tile by tile: each tile centres and scales its own operands (DESIGN section 4.6), so the result
    is held to the bound of its own tile's operands -- bounded here by the bound with the whole operands' magnitudes."""
    rng = np.random.default_rng(78)
    n, k, m, blk = 900, 600, 800, 200
    Af, Bf = rng.uniform(0, 1, (n, k)), rng.uniform(-1, 1, (k, m))
    A, B = to_blocks(Af, blk, random_mask(rng, 0.5)), to_blocks(Bf, blk, random_mask(rng, 0.5))
    with mb.MatfastSession(device=0, gemm_algo=3) as s:
        host = lambda ds: s.createHostDataset([mb.MatrixBlock(i, j, mb.DenseMatrix(v.numRows, v.numCols, v.values, v.isTransposed))  # noqa: E731
                                               for (i, j), v in sorted(ds.items())])
        C, st = _streamed(s, host(A), host(B), n, k, m, blk)
        assert C.isHost and st["stream_tiles"] >= 2 and st["tc_gemm_launches"] == 0
        assert st["kernel_launches"] >= st["stream_tiles"] * 5
        got = from_dataset(C)
    assert_same_dataset(got, O.matrix_multiply(A, n, k, B, k, m, blk), tol=1e-5)
    G = O.assemble(got, n, m, blk)
    # any tile's means are at most the largest |a| of the operand: U with |mu| <= max |a| covers every tile's own bound
    E = tf32_bound(Af, Bf, (float(np.abs(Af).max()), float(np.abs(Bf).max())))
    lim = E + fp64_dot_bound(Af, Bf)
    assert (np.abs(G - Af @ Bf) <= lim).all()
    pos = positions(rng, n, m, blk, 50, 100)
    for (i, j), x in zip(pos, exact_entries(Af, Bf, pos)):
        assert within(G[i, j], x, E[i, j]), (i, j)
    assert math.isfinite(float(G.max()))

"""GPU tests of the Ozaki-II Strassen route (option oz2_strassen, DESIGN section 4.1.3): one Strassen level per modulus must give
the plain route's result bit for bit, run where it is eligible (tc_strassen_jobs, 7/8 of the int8 operations) and nowhere else.
The small shapes use oz2_strassen = 2 (every eligible size); the default 1 takes the route from M, N, K >= 16384 on."""
import numpy as np
import pytest

import matrel_b200 as mb
from oracle import matrel_oracle as O
from tests.util import assert_same_dataset, from_dataset, to_dataset

pytestmark = pytest.mark.gpu

DEFAULTS = {"gemm_algo": 4, "crt_moduli": 0, "ozaki_scratch_mb": 0, "gemm_variant": -1, "oz2_ksplit": 0, "oz2_strassen": 2}


@pytest.fixture(scope="module")
def sess():
    s = mb.MatfastSession(device=0, gemm_algo=4)
    yield s
    s.stop()


def multiply(s, A, B, n, k, m, blk, **opts):
    for key, v in {**DEFAULTS, **opts}.items():
        s.set_option(key, v)
    try:
        s.reset_stats()
        got = from_dataset(to_dataset(s, A).matrixMultiply(n, k, to_dataset(s, B), k, m, blk))
        return got, s.stats()
    finally:
        for key, v in DEFAULTS.items():
            s.set_option(key, v)


def to_blocks(M, blk, tmask=lambda i, j: False):
    n, m = M.shape
    out = {}
    for i in range(-(-n // blk)):
        for j in range(-(-m // blk)):
            sub = M[i * blk:(i + 1) * blk, j * blk:(j + 1) * blk]
            if tmask(i, j):
                out[(i, j)] = O.DenseMatrix(sub.shape[0], sub.shape[1], np.ascontiguousarray(sub).reshape(-1), True)
            else:
                out[(i, j)] = O.DenseMatrix(sub.shape[0], sub.shape[1], np.ascontiguousarray(sub.T).reshape(-1), False)
    return out


def same_bits(got, ref):
    assert_same_dataset(got, {k: O.DenseMatrix(v.numRows, v.numCols, v.values) for k, v in ref.items()}, exact_storage=True)


def both_routes(s, A, B, n, k, m, blk, **opts):
    """The product with the route on and off; checks that the route ran once, on 7/8 of the int8 work, with the same bits."""
    plain, st0 = multiply(s, A, B, n, k, m, blk, oz2_strassen=0, **opts)
    got, st1 = multiply(s, A, B, n, k, m, blk, **opts)
    assert st0["tc_strassen_jobs"] == 0 and st1["tc_strassen_jobs"] == 1
    assert st0["tc_gemm_launches"] == 1 and st1["tc_gemm_launches"] == 1
    assert st1["tc_moduli"] == st0["tc_moduli"]
    assert st1["tc_int8_ops"] * 8 == st0["tc_int8_ops"] * 7
    same_bits(got, plain)
    return got


ELIGIBLE = [
    (2048, 2048, 2048, 512),     # square, 4 x 4 blocks
    (1024, 2048, 3072, 512),     # rectangular: 2 x 4 times 4 x 6 blocks
    (2048, 4096, 2048, 1024),    # blk 1024
    (2048, 2048, 2560, 256),     # blk 256: 8 x 8 times 8 x 10 blocks
]


@pytest.mark.parametrize("algo", [4, 0])
@pytest.mark.parametrize("n,k,m,blk", ELIGIBLE, ids=["%dx%dx%d-blk%d" % c for c in ELIGIBLE])
def test_strassen_route_is_bit_identical(sess, n, k, m, blk, algo):
    rng = np.random.default_rng(n + 3 * k + 7 * m + algo)
    Af, Bf = rng.uniform(-1.0, 1.0, (n, k)), rng.standard_normal((k, m)) * np.exp2(rng.integers(-20, 20, (1, m)))
    table = rng.random((16, 16)) < 0.5                          # row-major blocks mixed in, on both sides
    A, B = to_blocks(Af, blk, lambda i, j: bool(table[i, j])), to_blocks(Bf, blk, lambda i, j: bool(table[j, i]))
    got = both_routes(sess, A, B, n, k, m, blk, gemm_algo=algo)
    G, ref = O.assemble(got, n, m, blk), Af @ Bf
    assert np.max(np.abs(G - ref)) <= 1e-12 * np.max(np.abs(Af) @ np.abs(Bf))


def test_single_cta_kernel_and_ksplit_order(sess):
    rng = np.random.default_rng(5)
    n, blk = 2048, 512
    Af, Bf = rng.uniform(0.0, 1.0, (n, n)), rng.uniform(-1.0, 1.0, (n, n))
    A, B = to_blocks(Af, blk), to_blocks(Bf, blk, lambda i, j: (i + j) % 2 == 0)
    ref = both_routes(sess, A, B, n, n, n, blk)
    for opts in ({"gemm_variant": 2}, {"oz2_ksplit": 2}):
        got, st = multiply(sess, A, B, n, n, n, blk, **opts)
        assert st["tc_strassen_jobs"] == 1, opts
        same_bits(got, ref)


def test_full_size_product_over_several_plane_pieces(sess):
    """16384^2 with 1024-blocks: the 7 x 2048 sub-product tiles at 14 moduli need four 2 GiB plane pieces."""
    n, blk = 16384, 1024
    nb = n // blk
    keys = [(0, 0), (nb // 2, nb // 3), (nb - 1, nb - 1), (1, nb - 2), (nb - 1, 0), (nb // 2 - 1, nb // 2)]
    A, B = sess.rand(n, n, blk, 42), sess.rand(n, n, blk, 43)
    out, stats = {}, {}
    for mode in (0, 1):                                         # off, and the default
        for key, v in {**DEFAULTS, "oz2_strassen": mode}.items():
            sess.set_option(key, v)
        sess.reset_stats()
        C = A.matrixMultiply(n, n, B, n, n, blk)
        stats[mode] = sess.stats()
        out[mode] = [C.get_block(*key).values.copy() for key in keys]
        del C
    for key, v in DEFAULTS.items():
        sess.set_option(key, v)
    assert stats[0]["tc_strassen_jobs"] == 0 and stats[1]["tc_strassen_jobs"] == 1
    assert stats[1]["tc_int8_ops"] * 8 == stats[0]["tc_int8_ops"] * 7
    for x, y in zip(out[0], out[1]):
        assert np.array_equal(x, y)
    want = sum(A.get_block(keys[1][0], kk).to_numpy() @ B.get_block(kk, keys[1][1]).to_numpy() for kk in range(nb))
    assert np.max(np.abs(out[1][1] - want.reshape(-1, order="F"))) <= 1e-13 * np.max(np.abs(want))


def test_guard_outliers_in_every_quadrant(sess):
    """Range-guard outliers (2^-45 below their line maximum) in each quadrant of A and of B: recorded once, left out of every
    operand combination and added exactly by the fix-up, as on the plain route.  One outlier per row of A / column of B."""
    rng = np.random.default_rng(9)
    n, blk = 2048, 512
    Af, Bf = rng.uniform(0.25, 1.0, (n, n)), rng.uniform(1.0, 2.0, (n, n))
    Af[:, 0] = 1.0
    h = n // 2
    a_spots = [(5, 100), (300, h + 200), (h + 7, 20), (h + 500, h + 900)]         # (row, k) in quadrants 11, 12, 21, 22
    b_spots = [(50, 9), (h + 100, 400), (60, h + 6), (h + 1000, h + 800)]          # (k, column) in quadrants 11, 21, 12, 22
    for i, kk in a_spots:
        Af[i, kk] = rng.uniform(1.0, 2.0) * 2.0 ** -45
    for kk, j in b_spots:
        Bf[kk, j] = rng.uniform(1.0, 2.0) * 2.0 ** -45
    A, B = to_blocks(Af, blk, lambda i, j: (i + j) % 2 == 0), to_blocks(Bf, blk)
    got = both_routes(sess, A, B, n, n, n, blk, gemm_algo=0)
    G, ref = O.assemble(got, n, n, blk), Af @ Bf
    assert np.max(np.abs(G - ref) / (np.abs(Af) @ np.abs(Bf))) <= 1e-14


def test_inf_in_one_quadrant_takes_the_exact_fallback(sess):
    rng = np.random.default_rng(13)
    n, blk = 2048, 512
    Af, Bf = rng.uniform(-1.0, 1.0, (n, n)), rng.uniform(-1.0, 1.0, (n, n))
    Af[1500, 1700] = np.inf                                                         # quadrant A22
    A, B = to_blocks(Af, blk), to_blocks(Bf, blk)
    plain, _ = multiply(sess, A, B, n, n, n, blk, gemm_algo=0, oz2_strassen=0)
    got, _ = multiply(sess, A, B, n, n, n, blk, gemm_algo=0)
    same_bits(got, plain)
    G = O.assemble(got, n, n, blk)
    with np.errstate(invalid="ignore"):
        ref = Af @ Bf
    assert np.array_equal(np.isnan(G), np.isnan(ref)) and np.array_equal(G[np.isinf(ref)], ref[np.isinf(ref)])
    fin = np.isfinite(ref)
    assert np.max(np.abs(G[fin] - ref[fin])) <= 1e-12 * n


INELIGIBLE = [
    ("odd_block_count", 1536, 2048, 2048, 512, {}),             # 3 block rows
    ("odd_k_blocks", 2048, 1536, 2048, 512, {}),                # 3 k-blocks
    ("ragged_last_block", 2000, 2048, 2048, 512, {}),           # last block row 464 high
    ("quadrant_not_pair_aligned", 1024, 1024, 1280, 128, {}),   # N / 2 = 640 is no multiple of 256
    ("panel_budget", 2048, 2048, 2048, 512, {"ozaki_scratch_mb": 48}),   # plain residues 117 MB: 2 x 2 panels
]


@pytest.mark.parametrize("name,n,k,m,blk,opts", INELIGIBLE, ids=[c[0] for c in INELIGIBLE])
def test_ineligible_products_keep_the_plain_route(sess, name, n, k, m, blk, opts):
    rng = np.random.default_rng(len(name))
    Af, Bf = rng.uniform(-1.0, 1.0, (n, k)), rng.uniform(-1.0, 1.0, (k, m))
    A, B = to_blocks(Af, blk), to_blocks(Bf, blk)
    plain, st0 = multiply(sess, A, B, n, k, m, blk, oz2_strassen=0, **opts)
    got, st = multiply(sess, A, B, n, k, m, blk, **opts)
    assert st["tc_gemm_launches"] == 1 and st["tc_strassen_jobs"] == 0
    assert st["tc_int8_ops"] == st0["tc_int8_ops"]
    same_bits(got, plain)


def test_default_takes_the_route_from_16384_on(sess):
    rng = np.random.default_rng(29)
    n, blk = 2048, 512
    A, B = to_blocks(rng.uniform(-1.0, 1.0, (n, n)), blk), to_blocks(rng.uniform(-1.0, 1.0, (n, n)), blk)
    plain, _ = multiply(sess, A, B, n, n, n, blk, oz2_strassen=0)
    got, st = multiply(sess, A, B, n, n, n, blk, oz2_strassen=1)
    assert st["tc_gemm_launches"] == 1 and st["tc_strassen_jobs"] == 0
    same_bits(got, plain)


def test_absent_block_keeps_the_plain_route(sess):
    rng = np.random.default_rng(17)
    n, blk = 2048, 512
    Af, Bf = rng.uniform(-1.0, 1.0, (n, n)), rng.uniform(-1.0, 1.0, (n, n))
    A, B = to_blocks(Af, blk), to_blocks(Bf, blk)
    del A[(1, 2)]
    got, st = multiply(sess, A, B, n, n, n, blk)
    assert st["tc_gemm_launches"] == 1 and st["tc_strassen_jobs"] == 0


def test_gram_product_keeps_its_own_route(sess):
    rng = np.random.default_rng(19)
    n, blk = 2048, 512
    Af = rng.uniform(-1.0, 1.0, (n, n))
    dA = to_dataset(sess, to_blocks(Af, blk))
    for key, v in {**DEFAULTS, "gemm_algo": 0}.items():
        sess.set_option(key, v)
    try:
        sess.reset_stats()
        got = from_dataset(dA.t().matrixMultiply(n, n, dA, n, n, blk))
        st = sess.stats()
    finally:
        for key, v in DEFAULTS.items():
            sess.set_option(key, v)
    assert st["gram_blocks"] > 0 and st["tc_strassen_jobs"] == 0
    G = O.assemble(got, n, n, blk)
    assert np.max(np.abs(G - Af.T @ Af)) <= 1e-12 * n


def test_pipelined_multiply_keeps_the_plain_route(sess):
    import torch
    rng = np.random.default_rng(23)
    n, blk = 4096, 512
    Af, Bf = rng.uniform(-1.0, 1.0, (n, n)), rng.uniform(-1.0, 1.0, (n, n))
    A, B = to_blocks(Af, blk), to_blocks(Bf, blk)
    ref, _ = multiply(sess, A, B, n, n, n, blk, gemm_algo=0, oz2_strassen=0)
    pin = lambda x: mb.DenseMatrix(x.numRows, x.numCols, torch.from_numpy(x.values).pin_memory().numpy(), x.isTransposed)  # noqa: E731
    pA = [mb.MatrixBlock(i, j, pin(x)) for (i, j), x in A.items()]
    pB = [mb.MatrixBlock(i, j, pin(x)) for (i, j), x in B.items()]
    for key, v in {**DEFAULTS, "gemm_algo": 0}.items():
        sess.set_option(key, v)
    try:
        sess.reset_stats()
        dA, dB = sess.emptyDataset(), sess.emptyDataset()
        for t in range(n // blk):
            dA.put_blocks([b for b in pA if b.rid == t])
            dB.put_blocks([b for b in pB if b.cid == t])
        got = from_dataset(dA.matrixMultiply(n, n, dB, n, n, blk))
        st = sess.stats()
    finally:
        for key, v in DEFAULTS.items():
            sess.set_option(key, v)
    assert st["tc_gemm_launches"] == 1 and st["tc_strassen_jobs"] == 0
    same_bits(got, ref)

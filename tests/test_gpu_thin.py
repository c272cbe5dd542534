"""GPU tests of the matrix x thin-matrix route (DESIGN section 4.5.5): C = A X and C = X A with X of 2 to 8 dense columns (rows)
over dense (both layouts), CSC and CSR matrix blocks.

Every call asserts its route: `mv_pairs`, `mv_sparse_entries` and the exact kernel launch count (one launch, plus one pre-pass when
a pair is CSC in A X or sparse in X A), and no engine launch.  Every result is compared bit for bit with tests/thin_ref.py, with the
t width-1 products of the columns of X (rows for X A) run on the GPU, and with a second run."""
import numpy as np
import pytest

import matrel_b200 as mb
from oracle import matrel_oracle as O
from tests import matvec_ref as R
from tests import thin_ref as T
from tests.test_gpu_matvec import KINDS, csc_of, csr_of, dense, matrix_blocks, same_bits, vector_blocks
from tests.util import from_dataset, to_dataset, to_product_matrix

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sess():
    s = mb.MatfastSession(device=0)
    yield s
    s.stop()


def thin_blocks(x, blk, rowmajor):
    """The blocks of a k x t (A X) or t x k (X A) array, in one layout."""
    return {(i, j): dense(x[i * blk:(i + 1) * blk, j * blk:(j + 1) * blk], rowmajor)
            for i in range(-(-x.shape[0] // blk)) for j in range(-(-x.shape[1] // blk))}


def run(s, A, X, xa, n, k, t, blk, dA=None, dX=None):
    dA = dA if dA is not None else to_dataset(s, A)
    dX = dX if dX is not None else to_dataset(s, X)
    s.sync()
    s.reset_stats()
    ds = dX.matrixMultiply(t, k, dA, k, n, blk) if xa else dA.matrixMultiply(n, k, dX, k, t, blk)
    s.sync()
    return from_dataset(ds), s.stats()


def route_counts(A, X, xa):
    """(pairs, stored entries of their sparse blocks, launches) the route takes."""
    pairs = entries = 0
    prepass = False
    for key, a in A.items():
        for xkey in X:
            if (xkey[1] if xa else xkey[0]) != (key[0] if xa else key[1]):
                continue
            pairs += 1
            if R.is_sparse(a):
                entries += a.values.size
                prepass = prepass or xa or not a.isTransposed
    return pairs, entries, 1 + prepass


def full(blocks, rows, cols, blk):
    out = np.zeros((rows, cols))
    for (i, j), m in blocks.items():
        v = m.to_numpy() if hasattr(m, "to_numpy") else m
        out[i * blk:i * blk + v.shape[0], j * blk:j * blk + v.shape[1]] = v
    return out


def check(s, A, X, xa, n, k, t, blk, x=None, dA=None, dX=None, width1=True):
    """The route's result for A X / X A, checked against thin_ref, the t width-1 GPU products (x: the k x t / t x k array of X,
    when X is whole) and a second run."""
    got, st = run(s, A, X, xa, n, k, t, blk, dA, dX)
    pairs, entries, launches = route_counts(A, X, xa)
    assert (st["mv_pairs"], st["mv_sparse_entries"]) == (pairs, entries)
    assert st["kernel_launches"] == launches and st["gemm_launches"] == 0 and st["tc_gemm_launches"] == 0
    want = T.product(A, X, xa)
    assert sorted(got) == sorted(want)
    for key, v in want.items():
        g = got[key]
        assert isinstance(g, mb.DenseMatrix) and not g.isTransposed and (g.numRows, g.numCols) == v.shape, key
        assert same_bits(g.to_numpy(), v), (key, np.argwhere(~((g.to_numpy() == v) | (np.isnan(g.to_numpy()) & np.isnan(v))))[:8])
    again, _ = run(s, A, X, xa, n, k, t, blk, dA, dX)
    for key in got:
        assert np.array_equal(got[key].values.view(np.int64), again[key].values.view(np.int64)), key
    if width1 and x is not None:
        C = full(got, t if xa else n, n if xa else t, blk)
        for j in range(t):
            v = x[j, :] if xa else x[:, j]
            one, _ = run(s, A, vector_blocks(v, blk, xa), xa, n, k, 1, blk, dA)
            c = full(one, 1 if xa else n, n if xa else 1, blk).reshape(-1)
            assert same_bits(C[j, :] if xa else C[:, j], c), j
    return got


# ------------------------------------------------------------------------------------------------ widths, forms, kinds, densities
CASES = [(kind, 1.0) for kind in ("dense_col", "dense_row")] + \
        [(kind, d) for kind in ("csc", "csr", "mixed") for d in (0.0, 1e-4, 1e-2, 0.3, 1.0)]


@pytest.mark.parametrize("t", [2, 3, 5, 8])
@pytest.mark.parametrize("xa", [False, True], ids=["AX", "XA"])
@pytest.mark.parametrize("kind,density", CASES, ids=[f"{k}-{d:g}" for k, d in CASES])
def test_every_width_kind_and_density(sess, kind, density, xa, t):
    rng = np.random.default_rng(len(kind) * 100 + int(density * 1e4) + 10 * xa + t)
    n, k, blk = 700, 1000, 256                                    # ragged output and k-blocks
    A = matrix_blocks(rng, k if xa else n, n if xa else k, blk, kind, density)
    x = rng.uniform(-1, 1, (t, k) if xa else (k, t))
    X = thin_blocks(x, blk, rowmajor=(t + len(kind)) % 2 == 1)      # both layouts across the cases
    check(sess, A, X, xa, n, k, t, blk, x=x)


@pytest.mark.parametrize("t", [3, 8])
def test_thin_sides_from_dense_and_transposed(sess, t):
    """fromDense of a C-order array gives row-major blocks; its t() is the left side of X^T S."""
    from matrel_b200.dataset import sprand
    rng = np.random.default_rng(50 + t)
    n, blk = 4096, 1024
    S = sprand(sess, n, n, blk, 1e-2, 5, csr=(t == 3))
    A = from_dataset(S)
    x = np.ascontiguousarray(rng.uniform(-1, 1, (n, t)))
    dX = sess.fromDense(x, blk)
    X = from_dataset(dX)
    assert all(m.isTransposed for m in X.values())
    check(sess, A, X, False, n, n, t, blk, x=x, dA=S, dX=dX)
    dXt = dX.t()
    check(sess, A, from_dataset(dXt), True, n, n, t, blk, x=x.T, dA=S, dX=dXt)


# ------------------------------------------------------------------------------------------------ values and structure
def messy_sparse(rng, rows, cols, csr):
    """Unsorted lines, repeated positions, explicit zeros and -0.0, +-inf and NaN among the stored values."""
    nl, ni = (rows, cols) if csr else (cols, rows)
    ptr, idx, val = [0], [], []
    for _ in range(nl):
        c = rng.choice(ni, int(rng.integers(0, 6)), replace=False)
        if c.size and rng.random() < 0.5:
            c = np.append(c, c[0])
        v = rng.uniform(-1, 1, c.size)
        v[rng.random(c.size) < 0.1] = 0.0
        v[rng.random(c.size) < 0.1] = -0.0
        idx.extend(c.tolist())
        val.extend(v.tolist())
        ptr.append(len(idx))
    val = np.asarray(val)
    if val.size > 3:
        val[1], val[2], val[3] = np.inf, -np.inf, np.nan
    return O.SparseMatrix(rows, cols, np.asarray(ptr, np.int32), np.asarray(idx, np.int32), val, csr)


@pytest.mark.parametrize("xa", [False, True], ids=["AX", "XA"])
@pytest.mark.parametrize("fmt", ["csc", "csr", "dense_col", "dense_row"])
def test_non_finite_values_in_a_and_x(sess, fmt, xa):
    rng = np.random.default_rng(11 + xa + 2 * len(fmt))
    n, k, blk, t = 300, 400, 128, 5
    rows, cols = (k, n) if xa else (n, k)
    if fmt.startswith("cs"):
        A = {(i, j): messy_sparse(rng, min(blk, rows - i * blk), min(blk, cols - j * blk), fmt == "csr")
             for i in range(-(-rows // blk)) for j in range(-(-cols // blk))}
    else:
        A = matrix_blocks(rng, rows, cols, blk, fmt, 1.0)
        A[(0, 0)].values[[3, 77, 200]] = [np.inf, -np.inf, np.nan]
    x = rng.uniform(-1, 1, (t, k) if xa else (k, t))
    for j, c in ((0, 5), (2, 200), (4, 300)):                    # non-finite values in single columns of X (rows for X A)
        x[(j, c) if xa else (c, j)] = [np.inf, np.nan, -np.inf][j // 2]
    x[(1, 17) if xa else (17, 1)] = -0.0
    check(sess, A, thin_blocks(x, blk, xa), xa, n, k, t, blk, x=x)


@pytest.mark.parametrize("xa", [False, True], ids=["AX", "XA"])
def test_non_finite_x_where_nothing_is_stored(sess, xa):
    """A X never reads X where no entry is stored; X A gives NaN there, in that row of X only."""
    n, k, blk, t = 64, 64, 64, 4
    a = np.zeros((k, n) if xa else (n, k))
    if xa:
        a[:10, :] = 1.0
    else:
        a[:, :10] = 1.0
    x = np.ones((t, k) if xa else (k, t))
    x[(2, 40) if xa else (40, 2)] = np.inf                        # row / column 40 of A stores nothing
    for fmt in ("csc", "csr"):
        got = check(sess, {(0, 0): KINDS[fmt](a)}, thin_blocks(x, blk, False), xa, n, k, t, blk, x=x)[(0, 0)].to_numpy()
        if xa:
            assert np.isnan(got[2]).all() and np.isfinite(np.delete(got, 2, axis=0)).all()
        else:
            assert np.isfinite(got).all()


@pytest.mark.parametrize("xa", [False, True], ids=["AX", "XA"])
def test_missing_blocks(sess, xa):
    rng = np.random.default_rng(21 + xa)
    n, k, blk, t = 600, 900, 256, 6
    A = matrix_blocks(rng, k if xa else n, n if xa else k, blk, "mixed", 0.05)
    A[(1, 1)] = csc_of(np.zeros((256, 256)))                       # no stored entry
    del A[(0, 2) if not xa else (2, 0)]                            # an absent matrix block
    x = rng.uniform(-1, 1, (t, k) if xa else (k, t))
    X = thin_blocks(x, blk, False)
    del X[(1, 0) if not xa else (0, 1)]                            # k-block 1 has no X block: its pairs do not exist
    check(sess, A, X, xa, n, k, t, blk)


@pytest.mark.parametrize("xa", [False, True], ids=["AX", "XA"])
@pytest.mark.parametrize("kind", ["dense_col", "csc", "csr", "mixed"])
def test_blk_smaller_than_t(sess, kind, xa):
    """Output blocks 3 wide and a ragged 2-wide one: several block columns (rows) on the thin side."""
    rng = np.random.default_rng(61 + xa + len(kind))
    n, k, blk, t = 20, 17, 3, 8
    A = matrix_blocks(rng, k if xa else n, n if xa else k, blk, kind, 0.5)
    x = rng.uniform(-1, 1, (t, k) if xa else (k, t))
    check(sess, A, thin_blocks(x, blk, xa), xa, n, k, t, blk, x=x)


def test_both_sides_thin(sess):
    rng = np.random.default_rng(71)
    k, blk = 1000, 256
    x = rng.uniform(-1, 1, (5, k))
    y = rng.uniform(-1, 1, (k, 7))
    check(sess, thin_blocks(x, blk, True), thin_blocks(y, blk, False), False, 5, k, 7, blk, x=y)   # X Y with A = X
    check(sess, thin_blocks(y, blk, False), thin_blocks(x, blk, False), True, 7, k, 5, blk, x=x)    # the same product written X A


@pytest.mark.parametrize("xa", [False, True], ids=["AX", "XA"])
@pytest.mark.parametrize("kind,blk", [("csr", 8192), ("csc", 8192), ("dense_col", 4096), ("dense_row", 4096)])
def test_blocks_of_4096_and_8192_rows(sess, kind, blk, xa):
    rng = np.random.default_rng(blk + len(kind) + xa)
    n, k, t = blk + 300, blk + 200, 8
    density = 1e-3 if kind.startswith("cs") else 1.0
    A = matrix_blocks(rng, k if xa else n, n if xa else k, blk, kind, density)
    x = rng.uniform(-1, 1, (t, k) if xa else (k, t))
    check(sess, A, thin_blocks(x, blk, True), xa, n, k, t, blk, x=x, width1=False)


# ------------------------------------------------------------------------------------------------ route selection
def test_gemm_algo_selects_the_engine_for_dense_pairs(sess):
    rng = np.random.default_rng(31)
    n, k, blk, t = 520, 700, 256, 4
    Ad = matrix_blocks(rng, n, k, blk, "dense_col", 1.0)
    As = matrix_blocks(rng, n, k, blk, "csr", 0.02)
    x = rng.uniform(-1, 1, (k, t))
    X = thin_blocks(x, blk, False)
    routed = check(sess, Ad, X, False, n, k, t, blk)
    try:
        for algo in (1, 2, 3, 4):
            sess.set_option("gemm_algo", algo)
            got, st = run(sess, Ad, X, False, n, k, t, blk)
            assert st["mv_pairs"] == 0 and st["gemm_launches"] + st["tc_gemm_launches"] >= 1, algo
            assert sorted(got) == sorted(routed)
            for key, v in routed.items():
                assert np.allclose(got[key].to_numpy(), v.to_numpy(), rtol=0, atol=(1e-5 if algo == 3 else 1e-11) * k), (algo, key)
            check(sess, As, X, False, n, k, t, blk)                 # no dense x dense pair: the route under every algo
            mixed = dict(As)
            mixed[(0, 0)] = Ad[(0, 0)]
            _, st = run(sess, mixed, X, False, n, k, t, blk)
            assert st["mv_pairs"] == 0, algo
    finally:
        sess.set_option("gemm_algo", 0)


@pytest.mark.parametrize("xa", [False, True], ids=["AX", "XA"])
@pytest.mark.parametrize("t", [9, 16])
def test_wider_sides_keep_their_routes(sess, t, xa):
    rng = np.random.default_rng(80 + t + xa)
    n, k, blk = 600, 700, 256
    A = matrix_blocks(rng, k if xa else n, n if xa else k, blk, "mixed", 0.05)
    x = rng.uniform(-1, 1, (t, k) if xa else (k, t))
    got, st = run(sess, A, thin_blocks(x, blk, False), xa, n, k, t, blk)
    assert st["mv_pairs"] == 0
    Af = full(A, k if xa else n, n if xa else k, blk)
    want = x @ Af if xa else Af @ x
    bound = 1.01 * (k + 2) * 2.0 ** -53 * ((np.abs(x) @ np.abs(Af)) if xa else (np.abs(Af) @ np.abs(x)))   # exact-sum bound
    C = full(got, t if xa else n, n if xa else t, blk)
    assert np.all(np.abs(C - want) <= bound + 1e-300)


# ------------------------------------------------------------------------------------------------ streamed
@pytest.mark.parametrize("xa", [False, True], ids=["AX", "XA"])
def test_streamed_matches_resident_bit_for_bit(xa):
    rng = np.random.default_rng(41 + xa)
    n, k, blk, t = 4096 + 100, 3000, 1024, 8
    A = matrix_blocks(rng, k if xa else n, n if xa else k, blk, "mixed", 0.3)
    X = thin_blocks(rng.uniform(-1, 1, (t, k) if xa else (k, t)), blk, True)
    with mb.MatfastSession(device=0) as s:
        hA = s.createHostDataset([mb.MatrixBlock(i, j, to_product_matrix(m)) for (i, j), m in sorted(A.items())])
        want = check(s, A, X, xa, n, k, t, blk)
        s.set_option("stream_budget_mb", 40)
        try:
            got, st = run(s, A, X, xa, n, k, t, blk, dA=hA)
        finally:
            s.set_option("stream_budget_mb", 0)
        assert st["stream_tiles"] >= 2, st["stream_tiles"]
        assert st["mv_pairs"] == route_counts(A, X, xa)[0]
        assert sorted(got) == sorted(want)
        for key in want:
            assert np.array_equal(got[key].values.view(np.int64), want[key].values.view(np.int64)), key


# ------------------------------------------------------------------------------------------------ sprand at N = 131072
@pytest.mark.parametrize("csr", [True, False], ids=["csr", "csc"])
def test_sprand_n131072(sess, csr):
    """S X, t(S) X and X^T S at N = 131072, density 1e-4, blk 1024, t = 8, each checked in full against thin_ref computed from the
    fetched blocks.  X^T S densified every block before (128 GiB of images)."""
    from matrel_b200.dataset import sprand
    N, blk, t = 131072, 1024, 8
    S = sprand(sess, N, N, blk, 1e-4, 11, csr=csr)
    St = S.t()
    x = np.random.default_rng(5).uniform(-1, 1, (N, t))
    dX = sess.fromDense(x, blk)
    dXt = dX.t()
    X, Xt = from_dataset(dX), from_dataset(dXt)
    for M, xa in ((S, False), (St, False), (S, True)):
        check(sess, from_dataset(M), Xt if xa else X, xa, N, N, t, blk, dA=M, dX=dXt if xa else dX, width1=False)


def test_block_power_iteration_equals_width_one_iterations(sess):
    """10 steps of X <- 0.5 (S X) with t = 8 equal, bit for bit, 8 independent width-1 iterations."""
    from matrel_b200.dataset import sprand
    N, blk, t = 16384, 1024, 8
    S = sprand(sess, N, N, blk, 1e-3, 3, csr=False)
    x = np.random.default_rng(9).uniform(-1, 1, (N, t))
    V = sess.fromDense(x, blk)
    for _ in range(10):
        V = S.matrixMultiply(N, N, V, N, t, blk).multiplyScalar(0.5)
    got = V.toNumpy(N, t, blk)
    for j in range(t):
        v = sess.fromDense(np.ascontiguousarray(x[:, j:j + 1]), blk)
        for _ in range(10):
            v = S.matrixMultiply(N, N, v, N, 1, blk).multiplyScalar(0.5)
        assert same_bits(got[:, j], v.toNumpy(N, 1, blk).reshape(-1)), j

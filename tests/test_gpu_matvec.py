"""GPU tests of the matrix x vector route (DESIGN section 4.5.5): C = A x and C = x A over dense (both layouts), CSC and CSR matrix
blocks with dense vector blocks.

Every call asserts its route: `mv_pairs`, `mv_sparse_entries` and the exact kernel launch count (one launch, plus one pre-pass
when a pair is CSC in A x or sparse in x A).  Every result is compared bit for bit with tests/matvec_ref.py, whose order the
route fixes, and every case runs twice for identical bits."""
import numpy as np
import pytest

import matrel_b200 as mb
from oracle import matrel_oracle as O
from tests import matvec_ref as R
from tests.util import from_dataset, to_dataset, to_product_matrix

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sess():
    s = mb.MatfastSession(device=0)
    yield s
    s.stop()


# ------------------------------------------------------------------------------------------------ operands
def dense(a, rowmajor=False):
    a = np.asarray(a, dtype=np.float64)
    return O.DenseMatrix(a.shape[0], a.shape[1], np.ascontiguousarray(a if rowmajor else a.T).reshape(-1), rowmajor)


def csc_of(a):
    ptr, idx, val = [0], [], []
    for c in range(a.shape[1]):
        nz = np.flatnonzero(a[:, c])
        idx.extend(nz.tolist())
        val.extend(a[nz, c].tolist())
        ptr.append(len(idx))
    return O.SparseMatrix(a.shape[0], a.shape[1], np.asarray(ptr, np.int32), np.asarray(idx, np.int32), np.asarray(val), False)


def csr_of(a):
    t = csc_of(a.T)
    return O.SparseMatrix(a.shape[0], a.shape[1], t.colPtrs, t.rowIndices, t.values, True)


KINDS = {"dense_col": dense, "dense_row": lambda a: dense(a, True), "csc": csc_of, "csr": csr_of}
MIXED = ["dense_col", "csc", "dense_row", "csr"]


def matrix_blocks(rng, rows, cols, blk, kind, density):
    out = {}
    for i in range(-(-rows // blk)):
        for j in range(-(-cols // blk)):
            r, c = min(blk, rows - i * blk), min(blk, cols - j * blk)
            a = np.where(rng.random((r, c)) < density, rng.uniform(-1, 1, (r, c)), 0.0)
            out[(i, j)] = KINDS[MIXED[(i + j) % 4] if kind == "mixed" else kind](a)
    return out


def vector_blocks(x, blk, xa):
    k = x.size
    return {((0, b) if xa else (b, 0)): O.DenseMatrix(*((1, n) if xa else (n, 1)), x[b * blk:b * blk + n].copy())
            for b in range(-(-k // blk)) for n in [min(blk, k - b * blk)]}


# ------------------------------------------------------------------------------------------------ the checks
def multiply(s, A, X, xa, n, k, blk, dA=None, dX=None):
    dA = dA if dA is not None else to_dataset(s, A)
    dX = dX if dX is not None else to_dataset(s, X)
    s.sync()
    s.reset_stats()
    ds = dX.matrixMultiply(1, k, dA, k, n, blk) if xa else dA.matrixMultiply(n, k, dX, k, 1, blk)
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


def same_bits(g, w):
    g, w = np.asarray(g, dtype=np.float64), np.asarray(w, dtype=np.float64)
    both_nan = np.isnan(g) & np.isnan(w)
    return g.shape == w.shape and bool(np.all(both_nan | ((g.view(np.int64) == w.view(np.int64)) & ~np.isnan(g))))


def check(s, A, X, xa, n, k, blk, **kw):
    got, st = multiply(s, A, X, xa, n, k, blk, **kw)
    pairs, entries, launches = route_counts(A, X, xa)
    assert (st["mv_pairs"], st["mv_sparse_entries"]) == (pairs, entries)
    assert st["kernel_launches"] == launches and st["gemm_launches"] == 0 and st["tc_gemm_launches"] == 0
    want = R.product(A, X, xa)
    assert sorted(got) == sorted(want)
    for key, v in want.items():
        g = got[key]
        assert isinstance(g, mb.DenseMatrix) and not g.isTransposed
        assert (g.numRows, g.numCols) == ((1, v.size) if xa else (v.size, 1)), key
        assert same_bits(g.values, v), (key, np.flatnonzero(~((g.values == v) | (np.isnan(g.values) & np.isnan(v))))[:8])
    again, _ = multiply(s, A, X, xa, n, k, blk, **kw)
    for key in got:
        assert np.array_equal(got[key].values.view(np.int64), again[key].values.view(np.int64)), key
    return got


# ------------------------------------------------------------------------------------------------ forms, kinds, densities
CASES = [(kind, 1.0) for kind in ("dense_col", "dense_row")] + \
        [(kind, d) for kind in ("csc", "csr", "mixed") for d in (0.0, 1e-4, 1e-2, 0.3, 1.0)]


@pytest.mark.parametrize("xa", [False, True], ids=["Ax", "xA"])
@pytest.mark.parametrize("kind,density", CASES, ids=[f"{k}-{d:g}" for k, d in CASES])
def test_every_kind_and_density(sess, kind, density, xa):
    rng = np.random.default_rng(len(kind) * 100 + int(density * 1e4) + xa)
    n, k, blk = 700, 1000, 256                                    # ragged output and k-blocks
    A = matrix_blocks(rng, k if xa else n, n if xa else k, blk, kind, density)
    X = vector_blocks(rng.uniform(-1, 1, k), blk, xa)
    check(sess, A, X, xa, n, k, blk)


def test_dot_product(sess):
    rng = np.random.default_rng(3)
    k, blk = 1000, 256
    X = vector_blocks(rng.uniform(-1, 1, k), blk, True)            # 1 x k
    Y = vector_blocks(rng.uniform(-1, 1, k), blk, False)           # k x 1
    check(sess, X, Y, False, 1, k, blk)


# ------------------------------------------------------------------------------------------------ values and structure
def messy_sparse(rng, rows, cols, csr):
    """Unsorted lines, repeated positions, explicit zeros and -0.0, +-inf and NaN among the stored values."""
    nl, ni = (rows, cols) if csr else (cols, rows)
    ptr, idx, val = [0], [], []
    for _ in range(nl):
        c = rng.choice(ni, int(rng.integers(0, 6)), replace=False)
        if c.size and rng.random() < 0.5:
            c = np.append(c, c[0])                                # a repeat
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


@pytest.mark.parametrize("xa", [False, True], ids=["Ax", "xA"])
@pytest.mark.parametrize("fmt", ["csc", "csr"])
def test_messy_blocks_and_non_finite_values(sess, fmt, xa):
    rng = np.random.default_rng(11 + xa + 2 * (fmt == "csr"))
    n, k, blk = 300, 400, 128
    rows, cols = (k, n) if xa else (n, k)
    A = {(i, j): messy_sparse(rng, min(blk, rows - i * blk), min(blk, cols - j * blk), fmt == "csr")
         for i in range(-(-rows // blk)) for j in range(-(-cols // blk))}
    x = rng.uniform(-1, 1, k)
    x[[5, 200]] = [np.inf, np.nan]
    x[17] = -0.0
    check(sess, A, vector_blocks(x, blk, xa), xa, n, k, blk)


@pytest.mark.parametrize("xa", [False, True], ids=["Ax", "xA"])
def test_non_finite_x_where_nothing_is_stored(sess, xa):
    """A x never reads x where no entry is stored; x A gives NaN there, as the dense image does."""
    n, k, blk = 64, 64, 64
    a = np.zeros((k, n) if xa else (n, k))
    a[:, :10] = 1.0 if not xa else 0.0
    if xa:
        a[:10, :] = 1.0
    x = np.ones(k)
    x[40] = np.inf                                                 # row / column 40 of A stores nothing
    for fmt in ("csc", "csr"):
        got = check(sess, {(0, 0): KINDS[fmt](a)}, vector_blocks(x, blk, xa), xa, n, k, blk)
        v = got[(0, 0)].values
        assert np.isnan(v).all() if xa else np.isfinite(v).all()


@pytest.mark.parametrize("xa", [False, True], ids=["Ax", "xA"])
def test_missing_vector_blocks_and_empty_blocks(sess, xa):
    rng = np.random.default_rng(21 + xa)
    n, k, blk = 600, 900, 256
    A = matrix_blocks(rng, k if xa else n, n if xa else k, blk, "mixed", 0.05)
    A[(1, 1)] = csc_of(np.zeros((256, 256)))                       # no stored entry
    del A[(0, 2) if not xa else (2, 0)]                            # an absent matrix block
    if not xa:
        for kb in range(4):
            A.pop((2, kb), None)                                   # a whole block row absent: no output block
    X = vector_blocks(rng.uniform(-1, 1, k), blk, xa)
    del X[(1, 0) if not xa else (0, 1)]                            # k-block 1 has no vector block: its pairs do not exist
    got = check(sess, A, X, xa, n, k, blk)
    if not xa:
        assert sorted(got) == [(0, 0), (1, 0)]


@pytest.mark.parametrize("xa", [False, True], ids=["Ax", "xA"])
@pytest.mark.parametrize("kind,blk", [("csr", 8192), ("csc", 8192), ("dense_col", 4096), ("dense_row", 4096)])
def test_blocks_of_4096_and_8192_rows(sess, kind, blk, xa):
    rng = np.random.default_rng(blk + len(kind) + xa)
    n, k = blk + 300, blk + 200
    density = 1e-3 if kind.startswith("cs") else 1.0
    A = matrix_blocks(rng, k if xa else n, n if xa else k, blk, kind, density)
    check(sess, A, vector_blocks(rng.uniform(-1, 1, k), blk, xa), xa, n, k, blk)


# ------------------------------------------------------------------------------------------------ route selection
def test_gemm_algo_selects_the_engine_for_dense_pairs(sess):
    rng = np.random.default_rng(31)
    n, k, blk = 520, 700, 256
    Ad = matrix_blocks(rng, n, k, blk, "dense_col", 1.0)
    As = matrix_blocks(rng, n, k, blk, "csr", 0.02)
    X = vector_blocks(rng.uniform(-1, 1, k), blk, False)
    routed = check(sess, Ad, X, False, n, k, blk)
    try:
        for algo in (1, 2, 3, 4):
            sess.set_option("gemm_algo", algo)
            got, st = multiply(sess, Ad, X, False, n, k, blk)
            assert st["mv_pairs"] == 0 and st["gemm_launches"] + st["tc_gemm_launches"] >= 1, algo
            assert sorted(got) == sorted(routed)
            for key, v in routed.items():
                assert np.allclose(got[key].to_numpy(), v.to_numpy(), rtol=0, atol=(1e-5 if algo == 3 else 1e-11) * k), (algo, key)
            check(sess, As, X, False, n, k, blk)                    # no dense x dense pair: the route under every algo
            mixed = dict(As)
            mixed[(0, 0)] = Ad[(0, 0)]
            _, st = multiply(sess, mixed, X, False, n, k, blk)
            assert st["mv_pairs"] == 0, algo
    finally:
        sess.set_option("gemm_algo", 0)


def test_sparse_vector_blocks_keep_todays_routes(sess):
    rng = np.random.default_rng(32)
    n, k, blk = 300, 500, 128
    A = matrix_blocks(rng, n, k, blk, "dense_col", 1.0)
    X = {key: csc_of(np.where(rng.random((v.numRows, 1)) < 0.5, v.to_numpy(), 0.0))
         for key, v in vector_blocks(rng.uniform(-1, 1, k), blk, False).items()}
    got, st = multiply(sess, A, X, False, n, k, blk)
    assert st["mv_pairs"] == 0
    want = O.matrix_multiply(A, n, k, X, k, 1, blk)
    assert sorted(got) == sorted(want)
    assert np.allclose(O.assemble(got, n, 1, blk), O.assemble(want, n, 1, blk), rtol=0, atol=1e-11 * k)


# ------------------------------------------------------------------------------------------------ streamed
@pytest.mark.parametrize("xa", [False, True], ids=["Ax", "xA"])
def test_streamed_matches_resident_bit_for_bit(xa):
    rng = np.random.default_rng(41 + xa)
    n, k, blk = 4096 + 100, 3000, 1024
    A = matrix_blocks(rng, k if xa else n, n if xa else k, blk, "mixed", 0.3)
    X = vector_blocks(rng.uniform(-1, 1, k), blk, xa)
    with mb.MatfastSession(device=0) as s:
        rows = [mb.MatrixBlock(i, j, to_product_matrix(m)) for (i, j), m in sorted(A.items())]
        hA = s.createHostDataset(rows)
        want = check(s, A, X, xa, n, k, blk)
        s.set_option("stream_budget_mb", 40)
        try:
            got, st = multiply(s, A, X, xa, n, k, blk, dA=hA)
        finally:
            s.set_option("stream_budget_mb", 0)
        assert st["stream_tiles"] >= 2, st["stream_tiles"]
        assert st["mv_pairs"] == route_counts(A, X, xa)[0]
        assert sorted(got) == sorted(want)
        for key in want:
            assert np.array_equal(got[key].values.view(np.int64), want[key].values.view(np.int64)), key


# ------------------------------------------------------------------------------------------------ the planner's rewrites
def test_planner_rewrites_of_sparse_products_take_the_route(sess):
    from matrel_b200.dataset import sprand
    from matrel_b200.plan import LazyDataset, Planner
    n, blk = 2048, 512
    S = LazyDataset.of(sprand(sess, n, n, blk, 0.01, 7, csr=True))
    T = LazyDataset.of(sprand(sess, n, n, blk, 0.01, 8, csr=False))
    P = S.matrixMultiply(n, n, T, n, n, blk)
    queries = {"rowSum": P.rowSum(n, n), "colSum": P.colSum(n, n), "sum": P.sum(n, n),
               "project_row": P.project(n, n, blk, True, 700), "project_col": P.project(n, n, blk, False, 1500),
               "selection": P.selection(n, n, blk, 700, 1500)}
    for name, q in queries.items():
        sess.reset_stats()
        got = from_dataset(q.execute(planner=Planner(True)))
        assert sess.stats()["mv_pairs"] > 0, name
        want = from_dataset(q.execute(planner=Planner(False)))
        assert sorted(got) == sorted(want), name
        for key in want:
            g, w = got[key].to_numpy(), want[key].to_numpy()
            assert g.shape == w.shape and np.allclose(g, w, rtol=1e-12, atol=1e-12 * max(1.0, np.abs(w).max())), (name, key)


# ------------------------------------------------------------------------------------------------ sprand at N = 131072
@pytest.mark.parametrize("csr", [True, False], ids=["csr", "csc"])
def test_sprand_n131072(sess, csr):
    """S x, t(S) x and x^T S at N = 131072, density 1e-4, blk 1024, each checked in full against the reference computed from the
    fetched blocks.  x^T S densified every block before (128 GiB of images)."""
    from matrel_b200.dataset import sprand
    N, blk = 131072, 1024
    S = sprand(sess, N, N, blk, 1e-4, 11, csr=csr)
    St = S.t()
    x = np.random.default_rng(5).uniform(-1, 1, N)
    for name, M, xa in (("Sx", S, False), ("tSx", St, False), ("xS", S, True)):
        X = vector_blocks(x, blk, xa)
        dX = to_dataset(sess, X)
        A = from_dataset(M)
        check(sess, A, X, xa, N, N, blk, dA=M, dX=dX)

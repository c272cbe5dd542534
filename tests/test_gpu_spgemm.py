"""Sparse x sparse block products on the device (spgemm.cu): output blocks whose partials are all low-density sparse x sparse.

For inputs whose indices are sorted within each line the result must equal the JVM loops restated in tests/jvm_sparse_ref.py
exactly: block ids, formats, flags, index arrays and value bits (NaN compared as NaN).  Unsorted input: the same structure,
values within rounding."""
import numpy as np
import pytest
import scipy.sparse as sp

import matrel_b200 as mb
from matrel_b200.dataset import sprand
from oracle import matrel_oracle as O
from tests import jvm_sparse_ref as J
from tests.util import TIGHT_TOL, assert_same_dataset, from_dataset

pytestmark = pytest.mark.gpu


def _block(a, csr, shuffle_rng=None):
    """O.SparseMatrix (CSC, or CSR when csr) of the entries != 0 of the dense array a; shuffle_rng permutes each line's entries."""
    t = sp.csr_matrix(a) if csr else sp.csc_matrix(a)
    t.sort_indices()
    ptr, idx, val = t.indptr.copy(), t.indices.copy(), t.data.copy()
    if shuffle_rng is not None:
        for ln in range(len(ptr) - 1):
            perm = shuffle_rng.permutation(ptr[ln + 1] - ptr[ln]) + ptr[ln]
            idx[ptr[ln]:ptr[ln + 1]], val[ptr[ln]:ptr[ln + 1]] = idx[perm], val[perm]
    return O.SparseMatrix(a.shape[0], a.shape[1], ptr, idx, val, csr)


def _rand(rng, m, n, density):
    return np.where(rng.random((m, n)) < density, rng.uniform(0.5, 1.5, (m, n)) * rng.choice([-1.0, 1.0], (m, n)), 0.0)


def _blocks(rng, M, N, blk, density, csr, absent=(), shuffle=False):
    out = {}
    for i in range(-(-M // blk)):
        for j in range(-(-N // blk)):
            if (i, j) in absent:
                continue
            r, c = min(blk, M - i * blk), min(blk, N - j * blk)
            out[(i, j)] = _block(_rand(rng, r, c, density), csr(i, j), rng if shuffle else None)
    return out


def _dump(ds):
    out = {}
    for b in ds.collect():
        m = b.matrix
        s = isinstance(m, mb.SparseMatrix)
        out[(b.rid, b.cid)] = ("sparse" if s else "dense", bool(m.isTransposed), m.numRows, m.numCols, m.values.view(np.int64).copy(),
                               m.colPtrs.copy() if s else None, m.rowIndices.copy() if s else None)
    return out


def _assert_exact(got, want, values="bits"):
    assert sorted(got) == sorted(want)
    for k in want:
        g, w = got[k], want[k]
        assert g[:4] == w[:4], (k, g[:4], w[:4])
        for x, y in ((g[5], w[5]), (g[6], w[6])):
            assert (x is None) == (y is None) and (x is None or np.array_equal(x, y)), f"block {k}: index arrays differ"
        gv, wv = g[4].view(np.float64), w[4].view(np.float64)
        assert np.array_equal(np.isnan(gv), np.isnan(wv)), k
        fin = ~np.isnan(wv)
        if values == "bits":
            assert np.array_equal(g[4][fin], w[4][fin]), f"block {k}: values differ"
        else:
            np.testing.assert_allclose(gv[fin], wv[fin], rtol=1e-13, atol=1e-300)


def _run(s, A, B, M, K, N, blk):
    return s.createDataset(mb.MatrixBlock(i, j, _mb(m)) for (i, j), m in A.items()).matrixMultiply(
        M, K, s.createDataset(mb.MatrixBlock(i, j, _mb(m)) for (i, j), m in B.items()), K, N, blk)


def _mb(m):
    return mb.SparseMatrix(m.numRows, m.numCols, m.colPtrs, m.rowIndices, m.values, m.isTransposed)


def _want(A, B):
    return {k: J.dump(v) for k, v in J.multiply(A, B).items()}


FORMATS = {"csc_csc": (False, False), "csr_csr": (True, True), "csr_csc": (True, False), "csc_csr": (False, True)}


@pytest.mark.parametrize("pair", list(FORMATS))
@pytest.mark.parametrize("density", [0.004, 0.02, 0.06])
def test_format_pairs_bit_exact(session, pair, density):
    """The four loop nests over several k-blocks with ragged edges: chains that stay sparse (0.004) and chains that flip to dense
    mid-way (0.02 - 0.06); exact against the restated loops and within TIGHT_TOL of the oracle."""
    fa, fb = FORMATS[pair]
    rng = np.random.default_rng(int(density * 1000) + 7 * fa + fb)
    M, K, N, blk = 3 * 64 - 9, 5 * 64 - 30, 3 * 64 - 17, 64
    A = _blocks(rng, M, K, blk, density, lambda i, j: fa)
    B = _blocks(rng, K, N, blk, density, lambda i, j: fb)
    C = _run(session, A, B, M, K, N, blk)
    _assert_exact(_dump(C), _want(A, B))
    assert_same_dataset(from_dataset(C), O.matrix_multiply(A, M, K, B, K, N, blk), tol=TIGHT_TOL)


@pytest.mark.parametrize("density", [0.01, 0.04])
def test_mixed_format_chains(session, density):
    rng = np.random.default_rng(int(density * 100))
    M, blk = 4 * 48 - 5, 48
    A = _blocks(rng, M, M, blk, density, lambda i, j: (i * 3 + j) % 2 == 0)
    B = _blocks(rng, M, M, blk, density, lambda i, j: (i + 2 * j) % 3 == 0)
    C = _run(session, A, B, M, M, M, blk)
    _assert_exact(_dump(C), _want(A, B))
    assert_same_dataset(from_dataset(C), O.matrix_multiply(A, M, M, B, M, M, blk), tol=TIGHT_TOL)


@pytest.mark.parametrize("pair", list(FORMATS))
def test_absent_and_empty_blocks_stored_zeros_cancellation_and_nonfinite(session, pair):
    fa, fb = FORMATS[pair]
    rng = np.random.default_rng(3 + 2 * fa + fb)
    M, K, N, blk = 2 * 40 + 13, 3 * 40 + 1, 2 * 40 + 29, 40
    A = _blocks(rng, M, K, blk, 0.05, lambda i, j: fa, absent={(0, 1)})
    B = _blocks(rng, K, N, blk, 0.05, lambda i, j: fb, absent={(2, 0)})
    A[(1, 0)] = _block(np.zeros((40, 40)), fa)                          # a sparse block without entries
    # explicitly stored zeros, an Inf and a NaN
    a = _rand(rng, 40, 40, 0.05)
    a[3, 5] = np.inf
    a[7, 9] = np.nan
    blkA = _block(np.where(a == 0.0, 0.0, a), fa)
    vals = blkA.values.copy()
    vals[:2] = 0.0
    A[(0, 0)] = O.SparseMatrix(40, 40, blkA.colPtrs, blkA.rowIndices, vals, fa)
    # cancellation: block (1, 1) of C gets x and -x from its two k-blocks
    x = _rand(rng, 40, 40, 0.05)
    x[0, :] = 0.0
    x[0, 3], x[0, 11] = 0.7, -1.3                                       # row 0 stays at density 0.05 (a 1 x 40 block)
    A[(1, 1)] = _block(np.eye(40), fa)
    A[(1, 2)] = _block(np.zeros((40, 40)), fa)
    A[(1, 3)] = _block(_neg_eye(40, 1), fa)                            # the K edge block is one column wide
    B[(1, 1)] = _block(x, fb)
    B[(3, 1)] = _block(x[:1], fb)                                       # row 0 of C(1, 1): x[0] - x[0] == 0.0, dropped
    B[(3, 0)] = _block(-x[:1], fb)
    B[(3, 2)] = _block(np.zeros((1, 29)), fb)                          # the one-row / one-column edge blocks are set by hand:
    A[(0, 3)] = _block(np.zeros((40, 1)), fa)
    A[(2, 3)] = _block(_neg_eye(13, 1), fa)                            # random ones could exceed density 0.1
    C = _run(session, A, B, M, K, N, blk)
    want = _want(A, B)
    _assert_exact(_dump(C), want)
    row0 = np.asarray(J.multiply(A, B)[(1, 1)][1])[0]
    assert not np.any(row0[[3, 11]])


def _neg_eye(m, n):
    """m x n block with -1 at (0, 0) (the K edge block is one column wide)."""
    e = np.zeros((m, n))
    e[0, 0] = -1.0
    return e


@pytest.mark.parametrize("pair", list(FORMATS))
def test_unsorted_indices(session, pair):
    """Indices shuffled within every line: the structure is exact, the values within rounding."""
    fa, fb = FORMATS[pair]
    rng = np.random.default_rng(21 + 2 * fa + fb)
    M, blk = 3 * 50 - 11, 50
    A = _blocks(rng, M, M, blk, 0.06, lambda i, j: fa, shuffle=True)
    B = _blocks(rng, M, M, blk, 0.06, lambda i, j: fb, shuffle=True)
    _assert_exact(_dump(_run(session, A, B, M, M, M, blk)), _want(A, B), values="close")


@pytest.mark.parametrize("shape", [(3 * 64 - 5, 3 * 64, 2 * 64, 64, 0.03), (2300, 2300, 1000, 1000, 0.004),
                                   (4096, 2 * 4096, 700, 4096, 0.001), (8192, 600, 400, 8192, 0.004)],
                         ids=["blk64", "blk1000_ragged", "blk4096", "blk8192"])
@pytest.mark.parametrize("pair", ["csc_csc", "csc_csr", "csr_csr"])
def test_block_heights(session, shape, pair):
    """Output blocks from 64 to 8192 rows, ragged ones included (the per-warp accumulators move to global memory for tall
    blocks)."""
    M, K, N, blk, density = shape
    fa, fb = FORMATS[pair]
    rng = np.random.default_rng(blk + 3 * fa + fb)
    A = _blocks(rng, M, K, blk, density, lambda i, j: fa)
    B = _blocks(rng, K, N, blk, density, lambda i, j: fb)
    _assert_exact(_dump(_run(session, A, B, M, K, N, blk)), _want(A, B))


def test_csc_left_chains_are_deterministic(session):
    rng = np.random.default_rng(5)
    M, blk = 4 * 128, 128
    A = _blocks(rng, M, M, blk, 0.03, lambda i, j: False)
    B = _blocks(rng, M, M, blk, 0.03, lambda i, j: (i + j) % 2 == 1)
    first = _dump(_run(session, A, B, M, M, M, blk))
    _assert_exact(_dump(_run(session, A, B, M, M, M, blk)), first)


def _host_products(A, B):
    """sum over chain pairs and k of nnz(A(:, k)) * nnz(B(k, :)), from the stored structure."""
    total, pairs = 0, 0
    for (i, k), a in A.items():
        for (k2, j), b in B.items():
            if k2 != k:
                continue
            ca = np.bincount(a.rowIndices, minlength=a.numCols) if a.isTransposed else np.diff(a.colPtrs)
            rb = np.diff(b.colPtrs) if b.isTransposed else np.bincount(b.rowIndices, minlength=b.numRows)
            total += int(np.dot(ca.astype(np.int64), rb.astype(np.int64)))
            pairs += 1
    return total, pairs


def test_counters(session):
    rng = np.random.default_rng(8)
    M, blk = 3 * 64 - 9, 64
    A = _blocks(rng, M, M, blk, 0.03, lambda i, j: (i + j) % 2 == 0, absent={(1, 1)})
    B = _blocks(rng, M, M, blk, 0.03, lambda i, j: j == 1)
    session.reset_stats()
    _run(session, A, B, M, M, M, blk)
    st = session.stats()
    assert (st["spgemm_products"], st["spgemm_pairs"]) == _host_products(A, B)
    # sparse x dense: no chains
    dense = session.createDataset(mb.MatrixBlock(i, j, mb.DenseMatrix(m.numRows, m.numCols, np.ones(m.numRows * m.numCols)))
                                  for (i, j), m in B.items())
    session.createDataset(mb.MatrixBlock(i, j, _mb(m)) for (i, j), m in A.items()).matrixMultiply(M, M, dense, M, M, blk).collect()
    st = session.stats()
    assert st["spgemm_products"] == 0 and st["spgemm_pairs"] == 0


@pytest.mark.parametrize("csr_left", [True, False])
def test_capability_n65536(session, csr_left):
    """sprand A x B at N = 65536, blk 1024, density 1e-3: its dense images would take 96 GiB."""
    N, blk, d = 65536, 1024, 1e-3
    A = sprand(session, N, N, blk, d, 11, csr=csr_left)
    B = sprand(session, N, N, blk, d, 12, csr=True)
    session.reset_stats()
    C = A.matrixMultiply(N, N, B, N, N, blk)
    session.sync()
    st = session.stats()
    nb = N // blk
    rows = [(0, 0), (nb - 1, nb - 1), (7, 31), (40, 3), (63, 17)]
    blocks_a, blocks_b = {}, {}

    def get(ds, cache, key):
        if key not in cache:
            m = ds.get_block(*key)
            cache[key] = O.SparseMatrix(m.numRows, m.numCols, m.colPtrs, m.rowIndices, m.values, m.isTransposed)
        return cache[key]

    # the scalar products of the whole product, from the operands' structure
    ca = {}
    for i in range(nb):
        for k in range(nb):
            a = get(A, blocks_a, (i, k))
            ca[(i, k)] = (np.bincount(a.rowIndices, minlength=blk) if a.isTransposed else np.diff(a.colPtrs)).astype(np.int64)
    rb = {}
    for k in range(nb):
        for j in range(nb):
            b = get(B, blocks_b, (k, j))
            rb[(k, j)] = np.diff(b.colPtrs).astype(np.int64)
    total = 0
    for k in range(nb):
        sa = sum(ca[(i, k)] for i in range(nb))
        sb = sum(rb[(k, j)] for j in range(nb))
        total += int(np.dot(sa, sb))
    assert st["spgemm_products"] == total
    assert st["spgemm_pairs"] == nb ** 3
    for t, (i, j) in enumerate(rows):
        g = C.get_block(i, j)
        assert isinstance(g, mb.SparseMatrix)
        want = sum((_csr(blocks_a[(i, k)]) @ _csr(blocks_b[(k, j)]) for k in range(nb)), sp.csr_matrix((blk, blk)))
        got = sp.csc_matrix((g.values, g.rowIndices, g.colPtrs), shape=(blk, blk)) if not g.isTransposed else \
            sp.csr_matrix((g.values, g.rowIndices, g.colPtrs), shape=(blk, blk))
        w = want.tocsc()
        w.sort_indices()
        gc = got.tocsc()
        gc.sort_indices()
        assert np.array_equal(gc.indptr, w.indptr) and np.array_equal(gc.indices, w.indices)
        assert np.max(np.abs(gc.data - w.data) / np.abs(w.data)) <= 1e-12
        if t < 2:
            ref = J.multiply({(0, k): blocks_a[(i, k)] for k in range(nb)}, {(k, 0): blocks_b[(k, j)] for k in range(nb)})[(0, 0)]
            got_d = _dump_one(g)
            _assert_exact({0: got_d}, {0: J.dump(ref)})


def _csr(m):
    if m.isTransposed:
        return sp.csr_matrix((m.values, m.rowIndices, m.colPtrs), shape=(m.numRows, m.numCols))
    return sp.csc_matrix((m.values, m.rowIndices, m.colPtrs), shape=(m.numRows, m.numCols)).tocsr()


def _dump_one(m):
    s = isinstance(m, mb.SparseMatrix)
    return ("sparse" if s else "dense", bool(m.isTransposed), m.numRows, m.numCols, m.values.view(np.int64).copy(),
            m.colPtrs.copy() if s else None, m.rowIndices.copy() if s else None)


@pytest.mark.parametrize("density", [0.004, 0.03])
def test_streamed_matches_resident(density):
    rng = np.random.default_rng(int(density * 1000))
    M, K, N, blk = 1024, 768, 1024, 256
    A = _blocks(rng, M, K, blk, density, lambda i, j: (i + j) % 2 == 0)
    B = _blocks(rng, K, N, blk, density, lambda i, j: j % 2 == 1)
    with mb.MatfastSession(device=0) as s:
        rows = lambda d: [mb.MatrixBlock(i, j, _mb(m)) for (i, j), m in sorted(d.items())]
        want = _dump(s.createDataset(rows(A)).matrixMultiply(M, K, s.createDataset(rows(B)), K, N, blk))
        resident_products = s.stats()["spgemm_products"]
        for mbytes in (1, 2, 4, 8, 16, 32):
            s.set_option("stream_budget_mb", mbytes)
            try:
                C = s.createHostDataset(rows(A)).matrixMultiply(M, K, s.createHostDataset(rows(B)), K, N, blk)
                break
            except MemoryError:
                continue
        s.sync()
        st = s.stats()
        assert C.isHost and st["stream_tiles"] >= 2
        assert st["spgemm_products"] == resident_products
        _assert_exact(_dump(C), want)
        _assert_exact(want, _want(A, B))

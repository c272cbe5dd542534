"""GPU tests of the sparse Gram route (DESIGN section 4.1.2): C = A A^T and C = A^T A over the arrays A.t() shares with A, every
block of A sparse and every output block a sparse x sparse chain.  Square blocks below the diagonal come from their mirrors,
diagonal blocks from triangular chains.

Every case asserts:
  - exact equality with the JVM loops of tests/jvm_sparse_ref.py: ids, formats, flags, index arrays, value bits (NaN as NaN);
  - exact equality with the general route on a copy (the same blocks ingested again: other arrays, so the route is not taken);
  - C = C^T structurally and bit for bit, block (i, j) against block (j, i);
  - gram_blocks / gram_mirrored_blocks as the rule predicts, spgemm_pairs / spgemm_products against a host count of the work;
  - a second call giving the same result.
Shuffled lines take the general route through the fallback, with its bits.  Look-alikes leave both Gram counters at 0."""
import numpy as np
import pytest
import scipy.sparse as sp

import matrel_b200 as mb
from oracle import matrel_oracle as O
from tests import jvm_sparse_ref as J
from tests.test_gpu_spgemm import _assert_exact, _block, _blocks, _dump, _mb, _rand
from tests.util import to_dataset

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sess():
    s = mb.MatfastSession(device=0)
    yield s
    s.stop()


def _ds(s, blocks):
    return s.createDataset(mb.MatrixBlock(i, j, _mb(m)) for (i, j), m in blocks.items())


def _t(blocks):
    return {(j, i): O.SparseMatrix(m.numCols, m.numRows, m.colPtrs, m.rowIndices, m.values, not m.isTransposed)
            for (i, j), m in blocks.items()}


def _operands(blocks, kind):
    """The left and right block dicts of the product (the right one over the left one's arrays)."""
    return (blocks, _t(blocks)) if kind == "AAt" else (_t(blocks), blocks)


def _call(s, A, kind, shape, blk, right=None):
    m, n = shape
    R = A if right is None else right
    s.reset_stats()
    if kind == "AAt":
        C = A.matrixMultiply(m, n, R.t(), n, m, blk)
    else:
        C = A.t().matrixMultiply(n, m, R, m, n, blk)
    s.sync()
    return C, s.stats()


def _col_nnz(b):
    """Stored entries per column of a block."""
    return np.bincount(b.rowIndices, minlength=b.numCols) if b.isTransposed else np.diff(b.colPtrs)


def _row_nnz(b):
    return np.diff(b.colPtrs) if b.isTransposed else np.bincount(b.rowIndices, minlength=b.numRows)


def expected_work(Lb, Rb):
    """(gram_blocks, gram_mirrored_blocks, spgemm_pairs, spgemm_products) of the Gram route: every chain except square blocks
    below the diagonal; a diagonal chain performs, per column t of L(i, k), the products of its entries on rows r <= c."""
    shape = {}
    for (i, k), a in Lb.items():
        for (k2, j), b in Rb.items():
            if k2 == k:
                shape[(i, j)] = (a.numRows, b.numCols)
    computed = [ij for ij, (m, n) in shape.items() if not (ij[0] > ij[1] and m == n)]
    pairs = products = 0
    for (i, j) in computed:
        for (i2, k), a in Lb.items():
            if i2 != i or (k, j) not in Rb:
                continue
            pairs += 1
            ca = _col_nnz(a).astype(np.int64)
            if i == j:
                products += int(np.sum(ca * (ca + 1) // 2))
            else:
                products += int(np.dot(ca, _row_nnz(Rb[(k, j)]).astype(np.int64)))
    return len(computed), len(shape) - len(computed), pairs, products


def _assert_symmetric(got):
    for (i, j), g in got.items():
        h = got[(j, i)]
        assert g[2:4] == h[2:4][::-1], (i, j)
        if g[2] == g[3]:
            assert g[0] == h[0], (i, j)  # a square block and its mirror end in the same kind
        if "dense" in (g[0], h[0]):
            dg, dh = _dense_of(g), _dense_of(h).T
            assert np.array_equal(np.isnan(dg), np.isnan(dh)), (i, j)
            fin = ~np.isnan(dg)
            assert np.array_equal(dg.view(np.int64)[fin], dh.view(np.int64)[fin]), (i, j)
        else:
            a, b = _csc_of(g), _csc_of(h).T.tocsc()
            b.sort_indices()
            assert np.array_equal(a.indptr, b.indptr) and np.array_equal(a.indices, b.indices), (i, j)
            assert np.array_equal(bits(a.data), bits(b.data)), (i, j)


def bits(x):
    return np.where(np.isnan(x), np.nan, x).view(np.int64)


def _csc_of(d):
    kind, isT, m, n, vals, ptr, idx = d
    v = vals.view(np.float64)
    if isT:
        return sp.csr_matrix((v, idx, ptr), shape=(m, n)).tocsc()
    return sp.csc_matrix((v, idx, ptr), shape=(m, n))


def _dense_of(d):
    kind, isT, m, n, vals, ptr, idx = d
    v = vals.view(np.float64)
    if kind == "dense":
        return v.reshape(n, m).T.copy()
    return mb.SparseMatrix(m, n, ptr, idx, v, isT).to_numpy()


def check(s, blocks, kind, shape, blk, jvm=True):
    """Runs the Gram product of the block dict `blocks` (A, shape (m, n)) and all comparisons; returns the dump and stats."""
    A = _ds(s, blocks)
    copy = _ds(s, blocks)
    got_c, st = _call(s, A, kind, shape, blk)
    got = _dump(got_c)
    ref_c, st_ref = _call(s, A, kind, shape, blk, right=copy)
    assert (st_ref["gram_blocks"], st_ref["gram_mirrored_blocks"]) == (0, 0)
    _assert_exact(got, _dump(ref_c))
    Lb, Rb = _operands(blocks, kind)
    if jvm:
        _assert_exact(got, {k: J.dump(v) for k, v in J.multiply(Lb, Rb).items()})
    _assert_symmetric(got)
    gb, gm, pairs, products = expected_work(Lb, Rb)
    assert (st["gram_blocks"], st["gram_mirrored_blocks"]) == (gb, gm)
    assert (st["spgemm_pairs"], st["spgemm_products"]) == (pairs, products)
    again, _ = _call(s, A, kind, shape, blk)
    _assert_exact(_dump(again), got)
    return got, st


LAYOUTS = {"csc": lambda i, j: False, "csr": lambda i, j: True, "mixed": lambda i, j: (3 * i + j) % 2 == 0}


@pytest.mark.parametrize("kind", ["AAt", "AtA"])
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("density", [0.004, 0.02, 0.06])
def test_layouts_and_densities(sess, kind, layout, density):
    """Chains that stay sparse (0.004) and that flip to dense mid-way; ragged edges on both sides of A."""
    rng = np.random.default_rng(int(density * 1000) + len(layout) + len(kind))
    m, n, blk = 4 * 64 - 9, 5 * 64 - 30, 64
    check(sess, _blocks(rng, m, n, blk, density, LAYOUTS[layout]), kind, (m, n), blk)


@pytest.mark.parametrize("m,n,blk,density", [(3 * 40 + 7, 2 * 40 + 3, 40, 0.05), (5 * 100 - 37, 3 * 100, 100, 0.02),
                                             (2 * 1024 + 300, 1500, 1024, 0.003)], ids=["blk40", "blk100", "blk1024"])
def test_block_sizes_with_ragged_edges(sess, m, n, blk, density):
    """The ragged last block row gives non-square off-diagonal blocks: both of their chains are computed."""
    rng = np.random.default_rng(blk)
    got, st = check(sess, _blocks(rng, m, n, blk, density, LAYOUTS["mixed"]), "AAt", (m, n), blk)
    nb = -(-m // blk)
    assert st["gram_mirrored_blocks"] == (nb - 1) * (nb - 2) // 2 and st["gram_blocks"] == nb * (nb + 1) // 2 + nb - 1


@pytest.mark.parametrize("kind,csr", [("AAt", False), ("AtA", True)])
def test_single_block_2300(sess, kind, csr):
    rng = np.random.default_rng(23)
    got, st = check(sess, _blocks(rng, 2300, 2300, 2300, 0.002, lambda i, j: csr), kind, (2300, 2300), 2300)
    assert (st["gram_blocks"], st["gram_mirrored_blocks"]) == (1, 0)


@pytest.mark.parametrize("density", [0.0004, 0.004])
def test_single_block_8192(sess, density):
    """Accumulators in global memory; checked against the general route only (the JVM restatement is too slow here)."""
    rng = np.random.default_rng(81)
    m, n = 8192, 3000
    a = _rand(rng, m, n, density)
    check(sess, {(0, 0): _block(a, True)}, "AAt", (m, n), 8192, jvm=False)


def test_absent_and_empty_blocks(sess):
    rng = np.random.default_rng(4)
    m, n, blk = 4 * 48 - 5, 3 * 48 + 11, 48
    blocks = _blocks(rng, m, n, blk, 0.05, LAYOUTS["mixed"], absent={(0, 1), (2, 0), (3, 3)})
    blocks[(1, 1)] = _block(np.zeros((48, 48)), True)
    blocks[(2, 2)] = _block(np.zeros((48, 48)), False)
    check(sess, blocks, "AAt", (m, n), blk)
    check(sess, blocks, "AtA", (m, n), blk)


@pytest.mark.parametrize("kind", ["AAt", "AtA"])
def test_outer_product_of_one_k_block(sess, kind):
    rng = np.random.default_rng(6)
    m, n, blk = (5 * 64 - 3, 50, 64) if kind == "AAt" else (50, 5 * 64 - 3, 64)
    check(sess, _blocks(rng, m, n, blk, 0.05, LAYOUTS["mixed"]), kind, (m, n), blk)


@pytest.mark.parametrize("layout", ["csc", "csr"])
def test_stored_zeros_cancellation_and_nonfinite(sess, layout):
    rng = np.random.default_rng(9)
    m, n, blk = 2 * 40 + 13, 3 * 40, 40
    blocks = _blocks(rng, m, n, blk, 0.05, LAYOUTS[layout])
    f = LAYOUTS[layout](0, 0)
    a = _rand(rng, 40, 40, 0.05)
    a[0, :] = 0.0
    a[3, 5], a[7, 9], a[11, 2] = np.inf, np.nan, -np.inf
    b = _block(a, f)
    vals = b.values.copy()
    vals[np.nonzero(np.isfinite(vals))[0][:3]] = 0.0                 # explicitly stored zeros
    blocks[(0, 0)] = O.SparseMatrix(40, 40, b.colPtrs, b.rowIndices, vals, f)
    a10 = _rand(rng, 40, 40, 0.05)
    a10[0, :] = 0.0
    blocks[(1, 0)] = _block(a10, f)
    # rows 0 of block rows 0 and 1 share the column-0 entries of k-blocks 1 and 2 with opposite signs: C(0, 40) cancels to 0.0
    x, y = np.zeros((40, 40)), np.zeros((40, 40))
    x[0, 0], y[0, 0] = 1.0, 1.0
    blocks[(0, 1)] = _block(x, f)
    blocks[(1, 1)] = _block(y, f)
    x2, y2 = np.zeros((40, 40)), np.zeros((40, 40))
    x2[0, 0], y2[0, 0] = 1.0, -1.0
    blocks[(0, 2)] = _block(x2, f)
    blocks[(1, 2)] = _block(y2, f)
    got, _ = check(sess, blocks, "AAt", (m, n), blk)
    assert _dense_of(got[(0, 1)])[0, 0] == 0.0 and _dense_of(got[(1, 0)])[0, 0] == 0.0
    assert np.isnan(_dense_of(got[(0, 0)])).any()


@pytest.mark.parametrize("kind", ["AAt", "AtA"])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_shuffled_lines_take_the_fallback(sess, kind, layout):
    """Indices shuffled within every line: the general route's own bits (the mirror would differ in the last bits)."""
    rng = np.random.default_rng(31 + len(layout))
    m, n, blk = 3 * 50 - 11, 3 * 50, 50
    blocks = _blocks(rng, m, n, blk, 0.06, LAYOUTS[layout], shuffle=True)
    A, copy = _ds(sess, blocks), _ds(sess, blocks)
    got, st = _call(sess, A, kind, (m, n), blk)
    ref, _ = _call(sess, A, kind, (m, n), blk, right=copy)
    _assert_exact(_dump(got), _dump(ref))
    Lb, Rb = _operands(blocks, kind)
    _assert_exact(_dump(got), {k: J.dump(v) for k, v in J.multiply(Lb, Rb).items()}, values="close")
    # the stored lines of the left operand's CSR blocks are walked unconverted by the diagonal chains, so any such block falls
    # back; a left operand of CSC blocks only is walked through sorted conversions and keeps the route
    left_csc = (kind, layout) in (("AAt", "csc"), ("AtA", "csr"))
    if left_csc:
        assert st["gram_blocks"] > 0
    else:
        assert (st["gram_blocks"], st["gram_mirrored_blocks"]) == (0, 0)


def test_pipelined_ingest(sess):
    import torch
    rng = np.random.default_rng(41)
    m, n, blk = 4 * 64 - 7, 3 * 64, 64
    blocks = _blocks(rng, m, n, blk, 0.03, LAYOUTS["mixed"])
    pin = lambda x: mb.SparseMatrix(x.numRows, x.numCols, torch.from_numpy(x.colPtrs).pin_memory().numpy(),  # noqa: E731
                                    torch.from_numpy(x.rowIndices).pin_memory().numpy(),
                                    torch.from_numpy(x.values).pin_memory().numpy(), x.isTransposed)
    pb = [mb.MatrixBlock(i, j, pin(x)) for (i, j), x in blocks.items()]
    dA = sess.emptyDataset()
    for t in range(-(-m // blk)):
        dA.put_blocks([b for b in pb if b.rid == t])
    got, st = _call(sess, dA, "AAt", (m, n), blk)
    Lb, Rb = _operands(blocks, "AAt")
    _assert_exact(_dump(got), {k: J.dump(v) for k, v in J.multiply(Lb, Rb).items()})
    assert (st["gram_blocks"], st["gram_mirrored_blocks"]) == expected_work(Lb, Rb)[:2]


def test_under_every_gemm_algo(sess):
    rng = np.random.default_rng(12)
    m, n, blk = 3 * 64, 2 * 64, 64
    blocks = _blocks(rng, m, n, blk, 0.02, LAYOUTS["csr"])
    for algo in (1, 2, 3, 4):
        sess.set_option("gemm_algo", algo)
        try:
            check(sess, blocks, "AAt", (m, n), blk)
        finally:
            sess.set_option("gemm_algo", 0)


def test_look_alikes_keep_the_general_route(sess):
    rng = np.random.default_rng(51)
    m, n, blk = 3 * 64 - 5, 2 * 64 + 9, 64
    blocks = _blocks(rng, m, n, blk, 0.03, LAYOUTS["mixed"])
    A = _ds(sess, blocks)

    def counters(L, R, d=(n, m, m, n)):
        sess.reset_stats()
        L.matrixMultiply(d[0], d[1], R, d[2], d[3], blk)
        sess.sync()
        st = sess.stats()
        return st["gram_blocks"], st["gram_mirrored_blocks"]

    assert counters(A.t(), A) != (0, 0)                                   # the route itself
    assert counters(A.t(), A.multiplyScalar(1.0)) == (0, 0)              # a copy
    assert counters(A.t(), A.filter_blocks(2, 0)) == (0, 0)               # a subset of the blocks, same arrays
    L = A.t()
    b = blocks[(1, 1)]
    L.put_block(1, 1, mb.SparseMatrix(b.numCols, b.numRows, b.colPtrs.copy(), b.rowIndices.copy(), b.values.copy(),
                                      not b.isTransposed))
    assert counters(L, A) == (0, 0)                                       # one block replaced by a copy
    mixed = dict(blocks)
    mixed[(0, 0)] = O.DenseMatrix(64, 64, np.ascontiguousarray(_to_dense(blocks[(0, 0)]).T).reshape(-1))
    D = to_dataset(sess, mixed)
    assert counters(D.t(), D) == (0, 0)                                   # a dense block among sparse ones
    dense_blk = dict(blocks)
    dense_blk[(1, 0)] = _block(_rand(rng, 64, 64, 0.2), False)            # a block above density 0.1
    S = _ds(sess, dense_blk)
    assert counters(S.t(), S) == (0, 0)
    assert counters(A.t(), A.toHost()) == (0, 0)                          # a host-resident operand: the streamed multiply


def _to_dense(b):
    return mb.SparseMatrix(b.numRows, b.numCols, b.colPtrs, b.rowIndices, b.values, b.isTransposed).to_numpy()

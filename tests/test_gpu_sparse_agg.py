"""GPU tests of rowSum / colSum / trace / project / selection on sparse blocks, which run on their stored entries (sparse_agg.cu,
DESIGN section 4.5.4).

Every call asserts its route: `agg_sparse_blocks` / `agg_sparse_entries` and the exact kernel launch count, which does not grow
with the number of blocks and leaves no room for a densify launch.  Output entries whose blocks are all sparse, and every slice,
are compared bit for bit (NaN payloads aside) with tests/sparse_agg_ref.py; entries of lines that also have dense blocks are held
to the exact sum of their terms within 1.01 (t + 2) 2^-53 sum |terms|."""
from fractions import Fraction

import numpy as np
import pytest

import matrel_b200 as mb
from matrel_b200.dataset import sprand
from oracle import matrel_oracle as O
from tests import sparse_agg_ref as R
from tests.exact_ref import exact_dot
from tests.test_gpu_sparse_ew import blocks, seed, sparse_block
from tests.test_gpu_spmm_edges import dense
from tests.util import from_dataset, to_dataset

pytestmark = pytest.mark.gpu

AGG = {"row": "rowSum", "col": "colSum", "trace": "trace"}


@pytest.fixture(scope="module")
def sess():
    s = mb.MatfastSession(device=0)
    yield s
    s.stop()


def involved(op, ds):
    return {k: m for k, m in ds.items() if op != "trace" or k[0] == k[1]}


def assert_route(st, blocks_read, launches):
    sp = [m for m in blocks_read if R.is_sparse(m)]
    assert st["agg_sparse_blocks"] == len(sp)
    assert st["agg_sparse_entries"] == sum(m.values.size for m in sp)
    assert st["kernel_launches"] == launches, (st["kernel_launches"], launches)


def check_aggregate(s, op, ds, n, m, d=None):
    """One aggregate of the block dict ds (its dataset d, if already made) against the reference; returns the output."""
    d = d if d is not None else to_dataset(s, ds)
    s.sync()
    s.reset_stats()
    out = getattr(d, AGG[op])(n, m)
    st = s.stats()
    blk = involved(op, ds)
    launches = (1 if any(not R.is_sparse(x) for x in blk.values()) else 0) + \
               (2 if any(R.is_sparse(x) and x.values.size for x in blk.values()) else 0)
    assert_route(st, blk.values(), launches)
    got = from_dataset(out)
    want = R.aggregate(op, ds)
    assert sorted(got) == sorted(want)
    for key, (S, dense_blocks) in want.items():
        g = got[key].values
        if not dense_blocks:
            assert np.array_equal(R.bits(g), R.bits(S)), (op, key)
            continue
        for t in range(g.size):
            x = R.terms(op, ds, key, t)
            assert np.all(np.isfinite(x))
            assert abs(Fraction(float(g[t])) - exact_dot(x, np.ones(x.size))) <= Fraction(R.sum_bound(x)), (op, key, t)
    return got


def check_slices(s, ds, n, m, blk, rows, cols, d=None):
    """project of each row in rows and each column in cols, and selection of their crossings, against the reference."""
    d = d if d is not None else to_dataset(s, ds)
    got_all = []
    calls = [("project", True, i) for i in rows] + [("project", False, j) for j in cols] + \
            [("selection", i, j) for i in rows for j in cols]
    for call in calls:
        s.sync()
        s.reset_stats()
        if call[0] == "project":
            out = d.project(n, m, blk, call[1], call[2])
            want = R.project(ds, blk, call[1], call[2])
            bid, off = call[2] // blk, call[2] % blk
            read = [x for (r, c), x in ds.items()
                    if (r if call[1] else c) == bid and off < (x.numRows if call[1] else x.numCols)]
        else:
            out = d.selection(n, m, blk, call[1], call[2])
            want = R.selection(ds, blk, call[1], call[2])
            x = ds.get((call[1] // blk, call[2] // blk))
            read = [x] if want else []
        st = s.stats()
        assert_route(st, read, (1 if any(not R.is_sparse(x) for x in read) else 0) + (1 if any(R.is_sparse(x) for x in read) else 0))
        got = from_dataset(out)
        assert sorted(got) == sorted(want), call
        for key, w in want.items():
            assert got[key].numRows * got[key].numCols == w.size
            assert np.array_equal(R.bits(got[key].values), R.bits(w)), (call, key)
        got_all.append(got)
    return got_all


def all_ops(s, ds, n, m, blk, rows, cols):
    d = to_dataset(s, ds)
    for op in ("row", "col"):
        check_aggregate(s, op, ds, n, m, d)
    if n == m:
        check_aggregate(s, "trace", ds, n, m, d)
    check_slices(s, ds, n, m, blk, rows, cols, d)


FORMATS = {"csc": lambda i, j: "csc", "csr": lambda i, j: "csr", "mixed": lambda i, j: "csr" if (i + j) % 2 else "csc"}


@pytest.mark.parametrize("fmts", list(FORMATS))
@pytest.mark.parametrize("density", [0.0, 1e-4, 1e-2, 0.3, 1.0])
def test_formats_densities(sess, fmts, density):
    """All-sparse datasets with ragged edges (300 = 128 + 128 + 44): every output bit for bit."""
    rng = np.random.default_rng(seed(fmts, density))
    n, blk = 300, 128
    ds = blocks(n, blk, lambda r, c, i, j: sparse_block(rng, r, c, density, FORMATS[fmts](i, j)))
    all_ops(sess, ds, n, n, blk, rows=[0, 127, 200, 299], cols=[5, 128, 263])


@pytest.mark.parametrize("fmts", list(FORMATS))
def test_messy_blocks_and_determinism(sess, fmts):
    """Unsorted lines, repeated coordinates, explicit zeros, -0.0, +-Inf and NaN; two runs give the same bits."""
    rng = np.random.default_rng(seed("messy", fmts))
    n, blk = 200, 96
    ds = blocks(n, blk, lambda r, c, i, j: sparse_block(rng, r, c, 0.05, FORMATS[fmts](i, j), messy=True))
    d = to_dataset(sess, ds)
    for op in ("row", "col", "trace"):
        a = check_aggregate(sess, op, ds, n, n, d)
        b = check_aggregate(sess, op, ds, n, n, d)
        assert all(np.array_equal(R.bits(a[k].values), R.bits(b[k].values)) for k in a)
    rows = [int(r) for r in rng.integers(0, n, 4)]
    cols = [int(c) for c in rng.integers(0, n, 3)]
    check_slices(sess, ds, n, n, blk, rows, cols, d)


@pytest.mark.parametrize("fmts", list(FORMATS))
def test_dense_and_sparse_lines(sess, fmts):
    """Dense blocks (both layouts) next to sparse ones: mixed lines within the exact-sum bound, all-sparse lines bit for bit."""
    rng = np.random.default_rng(seed("mixed", fmts))
    n, blk = 260, 100

    def mk(r, c, i, j):
        if (i * 3 + j) % 4 == 0:
            return dense(rng.uniform(-1, 1, (r, c)) * 10.0 ** rng.integers(-3, 4), rowmajor=(i + j) % 2 == 1)
        return sparse_block(rng, r, c, 0.05, FORMATS[fmts](i, j))

    ds = blocks(n, blk, mk)
    all_ops(sess, ds, n, n, blk, rows=[0, 150, 259], cols=[99, 100, 210])


def test_empty_blocks_and_ragged_offsets(sess):
    """Empty sparse blocks give zero outputs; a row / column offset beyond a ragged block skips that block."""
    rng = np.random.default_rng(3)
    e_csc = O.SparseMatrix(64, 48, np.zeros(49, np.int32), np.zeros(0, np.int32), np.zeros(0), False)
    e_csr = O.SparseMatrix(64, 48, np.zeros(65, np.int32), np.zeros(0, np.int32), np.zeros(0), True)
    ds = {(0, 0): e_csc, (0, 1): e_csr, (1, 0): sparse_block(rng, 64, 48, 0.1, "csc"), (1, 1): e_csc}
    all_ops(sess, ds, 128, 96, 64, rows=[0, 70], cols=[3, 50])
    # block (0, 1) is 30 rows high and (1, 0) 20 columns wide: rows 30 .. 63 and columns 20 .. 63 skip them
    ds = {(0, 0): sparse_block(rng, 64, 64, 0.1, "csr"), (0, 1): sparse_block(rng, 30, 64, 0.1, "csc"),
          (1, 0): sparse_block(rng, 64, 20, 0.1, "csr"), (1, 1): sparse_block(rng, 64, 64, 0.1, "csc")}
    check_slices(sess, ds, 128, 128, 64, rows=[10, 40, 64], cols=[5, 30, 100])
    for op in ("row", "trace"):
        check_aggregate(sess, op, {k: v for k, v in ds.items() if k != (0, 1)}, 128, 128)


@pytest.mark.parametrize("rows", [4096, 8192])
def test_tall_blocks(sess, rows):
    """Outputs longer than the shared-memory accumulators: the warp accumulates in the block's partial slot in global memory."""
    rng = np.random.default_rng(rows)
    ds = {(0, 0): sparse_block(rng, rows, 40, 0.01, "csc"), (0, 1): sparse_block(rng, rows, 33, 0.02, "csc", messy=True),
          (0, 2): sparse_block(rng, rows, 20, 0.01, "csr")}
    check_aggregate(sess, "row", ds, rows, 93)
    check_slices(sess, ds, rows, 93, rows, rows=[0, rows - 1], cols=[7])
    dt = {(j, 0): sparse_block(rng, 40, rows, 0.01, "csr" if j else "csc", messy=j == 1) for j in range(3)}
    check_aggregate(sess, "col", dt, 120, rows)


def fetch(d):
    return {k: d.get_block(*k) for k in d.block_ids()}


def test_transposed_sprand(sess):
    n, blk = 2048, 256
    for csr in (True, False):
        A = sprand(sess, n, n, blk, 2e-3, 17, csr=csr).t()
        ds = fetch(A)
        assert all(R.is_sparse(m) and m.isTransposed != csr for m in ds.values())
        for op in ("row", "col", "trace"):
            check_aggregate(sess, op, ds, n, n, A)
        check_slices(sess, ds, n, n, blk, rows=[0, 1000], cols=[2047], d=A)


def test_more_than_65535_blocks(sess):
    """131072 sparse blocks of 4 x 4 in one call: one launch per pass."""
    n, blk = 1024, 4
    rng = np.random.default_rng(9)
    for csr in (True, False):
        A = sprand(sess, 2 * n, n, blk, 0.25, 101, csr=csr)
        for op, nout in (("row", 2 * n // blk), ("col", n // blk)):
            sess.sync()
            sess.reset_stats()
            out = getattr(A, AGG[op])(2 * n, n)
            st = sess.stats()
            assert st["agg_sparse_blocks"] == 2 * n * n // blk // blk
            assert st["kernel_launches"] == 2
            keys = {int(k) for k in rng.integers(0, nout, 4)} | {nout - 1}
            for k in keys:
                key = (k, 0) if op == "row" else (0, k)
                line = {(k, j): A.get_block(k, j) for j in range(n // blk)} if op == "row" else \
                       {(i, k): A.get_block(i, k) for i in range(2 * n // blk)}
                (S, _), = R.aggregate(op, line).values()
                assert np.array_equal(R.bits(out.get_block(*key).values), R.bits(S)), (op, key)


@pytest.mark.parametrize("csr", [True, False])
def test_sprand_131072(sess, csr):
    """N = 131072, blk 1024, density 1e-4: all five operators, whose dense images (128 GiB) could not be held; every output
    against the reference computed from the fetched blocks."""
    n, blk, nb = 131072, 1024, 128
    A = sprand(sess, n, n, blk, 1e-4, 5, csr=csr)
    ds = fetch(A)
    assert len(ds) == nb * nb
    for op in ("row", "col", "trace"):
        check_aggregate(sess, op, ds, n, n, A)
    check_slices(sess, ds, n, n, blk, rows=[0, 77777, n - 1], cols=[4242, n - 1], d=A)

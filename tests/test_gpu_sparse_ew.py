"""GPU tests of the element-wise joins with a sparse side (addElement / multiplyElement / divideElement), which run on the stored
entries of the sparse blocks (sparse_ew.cu, DESIGN section 4.5.3).

Every result block is compared bit for bit (NaN payloads aside) with tests/sparse_ew_ref.py, the reference's loops restated, and
every call asserts its route: `ew_sparse_pairs` / `ew_sparse_entries` and the exact kernel launch count, which does not grow with
the number of pairs and leaves no room for a densify launch."""
import zlib

import numpy as np
import pytest

import matrel_b200 as mb
from matrel_b200.dataset import sprand
from oracle import matrel_oracle as O
from tests import sparse_ew_ref as R
from tests.test_gpu_spmm_edges import dense, rand_csr
from tests.util import from_dataset, to_dataset

pytestmark = pytest.mark.gpu

FN = {"add": "addElement", "mul": "multiplyElement", "div": "divideElement"}


def seed(*key):
    return zlib.crc32(repr(key).encode())


@pytest.fixture(scope="module")
def sess():
    s = mb.MatfastSession(device=0)
    yield s
    s.stop()


@pytest.fixture(scope="module")
def sess_intended():
    s = mb.MatfastSession(device=0, compat_bugs=False)
    yield s
    s.stop()


# ------------------------------------------------------------------------------------------------ operands
def rand_csc(rng, rows, cols, density, sort=True, dups=0.0):
    t = rand_csr(rng, cols, rows, density, sort=sort, dups=dups)
    return O.SparseMatrix(rows, cols, t.colPtrs, t.rowIndices, t.values, False)


def spoil(rng, s, share=0.1, specials=(0.0, -0.0, np.inf, -np.inf, np.nan)):
    """The same block with a share of its stored values replaced by explicit zeros, -0.0 and non-finite values."""
    v = s.values.copy()
    pick = rng.random(v.size) < share
    v[pick] = rng.choice(np.asarray(specials), pick.sum())
    return O.SparseMatrix(s.numRows, s.numCols, s.colPtrs, s.rowIndices, v, s.isTransposed)


def sparse_block(rng, rows, cols, density, fmt, messy=False):
    kw = dict(sort=not messy, dups=0.3 if messy else 0.0)
    s = rand_csc(rng, rows, cols, density, **kw) if fmt == "csc" else rand_csr(rng, rows, cols, density, **kw)
    return spoil(rng, s) if messy else s


def blocks(n, blk, make):
    nb = -(-n // blk)
    return {(i, j): make(min(blk, n - i * blk), min(blk, n - j * blk), i, j) for i in range(nb) for j in range(nb)}


# ------------------------------------------------------------------------------------------------ the reference and the route
def expected(op, A, B, compat=True):
    out = {}
    for key in set(A) | set(B):
        a, b = A.get(key), B.get(key)
        if a is None or b is None:
            if op == "add":
                out[key] = a if b is None else b
            continue
        da, db = isinstance(a, O.DenseMatrix), isinstance(b, O.DenseMatrix)
        if not da and not db:
            out[key] = R.sparse_sparse(op, a, b)
        elif da and not db:
            out[key] = R.dense_sparse(op, a, b, False)
        elif db and not da:
            out[key] = R.dense_sparse(op, b, a, not (op == "div" and compat))
        else:
            out[key] = None  # dense (+) dense: not this file's subject
    return out


def launches(A, B, want):
    """Kernel launches of the join: sptrans (4) when a sparse (+) sparse pair has a CSR side, the count pass, a scan when a result
    is sparse, the fill pass; one batched ew launch for dense pairs and a scatter when a dense (+) sparse pair stores entries."""
    spsp = [k for k in A if k in B and not isinstance(A[k], O.DenseMatrix) and not isinstance(B[k], O.DenseMatrix)]
    other = [k for k in A if k in B and k not in spsp]
    n = 0
    if spsp:
        n += 2 + (4 if any(A[k].isTransposed or B[k].isTransposed for k in spsp) else 0)
        n += 1 if any(want[k][0] == R.CSC for k in spsp) else 0
    if other:
        n += 1
        if any(not isinstance(x, O.DenseMatrix) and x.values.size for k in other for x in (A[k], B[k])):
            n += 1
    return n


def run(s, op, A, B, compat=True, check_keys=None):
    dA, dB = to_dataset(s, A), to_dataset(s, B)
    s.sync()
    s.reset_stats()
    dC = getattr(dA, FN[op])(1, 1, dB, 1, 1, 1)
    st = s.stats()
    want = expected(op, A, B, compat)
    pairs = [k for k in A if k in B and not (isinstance(A[k], O.DenseMatrix) and isinstance(B[k], O.DenseMatrix))]
    assert st["ew_sparse_pairs"] == len(pairs)
    assert st["ew_sparse_entries"] == sum(x.values.size for k in pairs for x in (A[k], B[k]) if not isinstance(x, O.DenseMatrix))
    assert st["kernel_launches"] == launches(A, B, want), (st["kernel_launches"], launches(A, B, want))
    got = from_dataset(dC)
    assert sorted(got) == sorted(k for k in want)
    for key in (check_keys if check_keys is not None else want):
        w = want[key]
        if w is None or not isinstance(w, tuple):
            continue
        R.assert_block(got[key], w, key)
    return got


def dump(got):
    return {k: (type(m).__name__, R.bits(m.values).tobytes(), None if not hasattr(m, "colPtrs") else np.asarray(m.colPtrs).tobytes())
            for k, m in got.items()}


# ------------------------------------------------------------------------------------------------ cases
FORMATS = {"csc": lambda i, j: ("csc", "csc"), "csr": lambda i, j: ("csr", "csr"),
           "mixed": lambda i, j: (("csr", "csc") if (i + j) % 2 else ("csc", "csr"))}


@pytest.mark.parametrize("op", ["add", "mul", "div"])
@pytest.mark.parametrize("fmts", list(FORMATS))
@pytest.mark.parametrize("density", [0.02, 0.9])
def test_ops_formats_densities(sess, op, fmts, density):
    """Ragged edge blocks (300 = 128 + 128 + 44), results on both sides of the output rule."""
    rng = np.random.default_rng(seed(op, fmts, density))
    n, blk = 300, 128
    A = blocks(n, blk, lambda r, c, i, j: sparse_block(rng, r, c, density, FORMATS[fmts](i, j)[0]))
    B = blocks(n, blk, lambda r, c, i, j: sparse_block(rng, r, c, density, FORMATS[fmts](i, j)[1]))
    got = run(sess, op, A, B)
    if op != "div":  # divide is NaN wherever nothing is stored: dense
        assert {type(m).__name__ for m in got.values()} == ({"SparseMatrix"} if density < 0.1 else {"DenseMatrix"})


@pytest.mark.parametrize("op", ["add", "mul", "div"])
@pytest.mark.parametrize("fmts", list(FORMATS))
def test_unsorted_repeats_zeros_nonfinite(sess, op, fmts):
    """Unsorted lines, repeated coordinates, explicit zeros, -0.0, +-Inf and NaN on either side, stored or facing an absent entry."""
    rng = np.random.default_rng(seed("messy", op, fmts))
    n, blk = 200, 96
    A = blocks(n, blk, lambda r, c, i, j: sparse_block(rng, r, c, 0.05, FORMATS[fmts](i, j)[0], messy=True))
    B = blocks(n, blk, lambda r, c, i, j: sparse_block(rng, r, c, 0.05, FORMATS[fmts](i, j)[1], messy=True))
    got = run(sess, op, A, B)
    assert dump(got) == dump(run(sess, op, A, B))  # determinism: the same bits twice


@pytest.mark.parametrize("op", ["add", "mul", "div"])
def test_empty_blocks_and_one_sided(sess, op):
    rng = np.random.default_rng(7)
    empty_csc = O.SparseMatrix(64, 48, np.zeros(49, np.int32), np.zeros(0, np.int32), np.zeros(0), False)
    empty_csr = O.SparseMatrix(64, 48, np.zeros(65, np.int32), np.zeros(0, np.int32), np.zeros(0), True)
    A = {(0, 0): empty_csc, (0, 1): empty_csr, (1, 0): sparse_block(rng, 64, 48, 0.1, "csc"), (1, 1): empty_csc,
         (2, 2): sparse_block(rng, 64, 48, 0.1, "csr")}
    B = {(0, 0): empty_csc, (0, 1): sparse_block(rng, 64, 48, 0.1, "csc"), (1, 0): empty_csr, (1, 1): empty_csr,
         (3, 3): sparse_block(rng, 64, 48, 0.1, "csc")}
    run(sess, op, A, B)


@pytest.mark.parametrize("rows", [4096, 8192])
@pytest.mark.parametrize("op", ["add", "mul"])
def test_tall_blocks(sess, rows, op):
    """Blocks taller than the shared-memory accumulators: the per-warp accumulators live in global scratch."""
    rng = np.random.default_rng(rows)
    A = {(0, 0): sparse_block(rng, rows, 40, 0.01, "csc"), (0, 1): sparse_block(rng, rows, 33, 0.02, "csr", messy=True)}
    B = {(0, 0): sparse_block(rng, rows, 40, 0.01, "csc", messy=True), (0, 1): sparse_block(rng, rows, 33, 0.02, "csc")}
    run(sess, op, A, B)


@pytest.mark.parametrize("op", ["add", "mul", "div"])
@pytest.mark.parametrize("rowmajor", [False, True])
@pytest.mark.parametrize("compat", [True, False])
def test_dense_sparse(sess, sess_intended, op, rowmajor, compat):
    """dense (+) sparse in both orders, both layouts of the dense side, with and without defect B4's divide swap."""
    s = sess if compat else sess_intended
    rng = np.random.default_rng(seed(op, rowmajor, compat))
    n, blk = 250, 100

    def dblock(r, c, i, j):
        a = rng.uniform(-1, 1, (r, c))
        a[rng.random((r, c)) < 0.02] = rng.choice([0.0, -0.0, np.inf, -np.inf, np.nan], 1)[0]
        return dense(a, rowmajor)

    def sblock(r, c, i, j):
        return sparse_block(rng, r, c, 0.05, "csr" if (i + 2 * j) % 3 == 0 else "csc", messy=(i + j) % 2 == 1)

    D, S = blocks(n, blk, dblock), blocks(n, blk, sblock)
    run(s, op, D, S, compat)
    got = run(s, op, S, D, compat)
    assert all(type(m).__name__ == "DenseMatrix" and not m.isTransposed for m in got.values())


def test_launches_do_not_grow_with_pairs(sess):
    rng = np.random.default_rng(11)
    mk = lambda r, c, i, j: sparse_block(rng, r, c, 0.01, "csr" if i == j else "csc")
    counts = []
    for n in (64, 640):
        A, B = blocks(n, 64, mk), blocks(n, 64, mk)
        dA, dB = to_dataset(sess, A), to_dataset(sess, B)
        sess.sync()
        sess.reset_stats()
        dA.addElement(n, n, dB, n, n, 64)
        counts.append(sess.stats()["kernel_launches"])
    assert counts[0] == counts[1] == 4 + 3, counts


def test_more_than_65535_pairs(sess):
    """131072 pairs of 4 x 4 sprand blocks in one call: the persistent grid covers them all."""
    n, blk = 1024, 4
    for csr in (True, False):
        A = sprand(sess, 2 * n, n, blk, 0.25, 101, csr=csr)
        B = sprand(sess, 2 * n, n, blk, 0.25, 202, csr=csr)
        sess.sync()
        sess.reset_stats()
        C = A.multiplyElement(2 * n, n, B, 2 * n, n, blk)
        st = sess.stats()
        assert st["ew_sparse_pairs"] == 2 * n * n // blk // blk
        assert st["kernel_launches"] == (4 if csr else 0) + 3
        rng = np.random.default_rng(5)
        keys = [(int(r), int(c)) for r, c in zip(rng.integers(0, 2 * n // blk, 300), rng.integers(0, n // blk, 300))]
        keys += [(2 * n // blk - 1, n // blk - 1 - t) for t in range(20)]   # pairs past 65535
        for k in keys:
            a, b = A.get_block(*k), B.get_block(*k)
            R.assert_block(C.get_block(*k), R.sparse_sparse("mul", a, b), k)


@pytest.mark.parametrize("csr", [True, False])
def test_sprand_131072(sess, csr):
    """N = 131072, blk 1024, density 1e-4: sums and Hadamard products whose dense images (128 GiB per operand) could not be held.
    Every block's format and structure is checked; sampled blocks bit for bit."""
    n, blk, nb = 131072, 1024, 128
    A = sprand(sess, n, n, blk, 1e-4, 1, csr=csr)
    B = sprand(sess, n, n, blk, 1e-4, 2, csr=csr)
    rng = np.random.default_rng(3)
    sample = {(int(r), int(c)) for r, c in zip(rng.integers(0, nb, 6), rng.integers(0, nb, 6))} | {(nb - 1, nb - 1)}
    for op in ("add", "mul"):
        sess.sync()
        sess.reset_stats()
        C = getattr(A, FN[op])(n, n, B, n, n, blk)
        st = sess.stats()
        assert st["ew_sparse_pairs"] == nb * nb
        assert st["kernel_launches"] == (4 if csr else 0) + 3
        first = (op == "add")
        for rid, cid in C.block_ids():
            c = C.get_block(rid, cid)
            a, b = A.get_block(rid, cid), B.get_block(rid, cid)
            assert type(c).__name__ == "SparseMatrix" and not c.isTransposed
            # sprand values are in (0, 1) and its coordinates distinct: the kept entries are the union (add) / intersection (mul)
            codes = []
            for s in (a, b):
                line = np.repeat(np.arange(len(s.colPtrs) - 1), np.diff(s.colPtrs))
                r, cc = (line, s.rowIndices) if s.isTransposed else (s.rowIndices, line)
                codes.append(cc.astype(np.int64) * blk + r)
            want = np.union1d(*codes) if first else np.intersect1d(*codes)
            cl = np.repeat(np.arange(blk), np.diff(c.colPtrs))
            assert np.array_equal(cl.astype(np.int64) * blk + c.rowIndices, want), (rid, cid)
            if (rid, cid) in sample:
                R.assert_block(c, R.sparse_sparse(op, a, b), (rid, cid))
        del C

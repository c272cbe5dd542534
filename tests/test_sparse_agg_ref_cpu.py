"""CPU checks of tests/sparse_agg_ref.py: the golden aggregates and slices, the oracle's intended reductions on data without
repeats, and hand-worked blocks for repeats, unsorted lines, -0.0 and non-finite values."""
import json
import os

import numpy as np

from oracle import matrel_oracle as O
from tests import sparse_agg_ref as R

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
NAN, INF = float("nan"), float("inf")


def csc(m, n, ptr, idx, val):
    return O.SparseMatrix(m, n, np.asarray(ptr, np.int32), np.asarray(idx, np.int32), np.asarray(val, np.float64), False)


def csr(m, n, ptr, idx, val):
    return O.SparseMatrix(m, n, np.asarray(ptr, np.int32), np.asarray(idx, np.int32), np.asarray(val, np.float64), True)


def as_csr(a):
    """The entries of an m x n array (!= 0) as a CSR block, columns ascending in each row."""
    t = O.DenseMatrix(a.shape[1], a.shape[0], np.ascontiguousarray(a).reshape(-1)).toSparse()  # CSC of a^T = CSR of a
    return csr(a.shape[0], a.shape[1], t.colPtrs, t.rowIndices, t.values)


def same(a, b):
    return np.array_equal(R.bits(a), R.bits(b))


def loop_partial(op, s):
    """Rule 1 as the reference's loops: line by line, entry by entry, one add each."""
    n = s.numRows if op == "row" else s.numCols
    out = [0.0] * (1 if op == "trace" else n)
    for line in range(len(s.colPtrs) - 1):
        for e in range(s.colPtrs[line], s.colPtrs[line + 1]):
            i, v = int(s.rowIndices[e]), float(s.values[e])
            r, c = (line, i) if s.isTransposed else (i, line)
            if op == "trace":
                if r == c:
                    out[0] = out[0] + v
            else:
                t = r if op == "row" else c
                out[t] = out[t] + v
    return np.array(out)


def messy(rng, m, n, nnz, transposed):
    """Unsorted lines with repeats, explicit zeros, -0.0 and non-finite values; values spread over many binades."""
    nl, ni = (m, n) if transposed else (n, m)
    counts = rng.multinomial(nnz, np.ones(nl) / nl)
    idx = rng.integers(0, ni, nnz)
    idx[1::7] = idx[::7][:idx[1::7].size]  # repeats
    val = rng.standard_normal(nnz) * 10.0 ** rng.integers(-8, 9, nnz)
    val[rng.random(nnz) < 0.05] = rng.choice([0.0, -0.0, INF, -INF, NAN], 1)[0]
    ptr = np.concatenate([[0], np.cumsum(counts)])
    return (csr if transposed else csc)(m, n, ptr, idx, val)


def test_add_at_is_storage_order():
    rng = np.random.default_rng(1)
    for transposed in (False, True):
        for _ in range(5):
            s = messy(rng, 37, 23, 400, transposed)
            for op in ("row", "col", "trace"):
                assert same(R.partial(op, s), loop_partial(op, s)), (op, transposed)


def test_golden_basic_matrix_ops():
    g = json.load(open(os.path.join(GOLDEN, "basic_matrix_ops.json")))
    e = g["expected"]

    def mk(v):
        if v["type"] == "dense":
            return O.DenseMatrix(v["numRows"], v["numCols"], v["values"])
        return csc(v["numRows"], v["numCols"], v["colPtrs"], v["rowIndices"], v["values"])

    blocks = {k: mk(v) for k, v in g["blocks"].items()}
    mat2 = {(r, c): blocks[n] for r, c, n in g["mat2"]}
    assert not isinstance(mat2[(1, 1)], O.DenseMatrix)  # block (1, 1) is sparse
    got = []
    for key, (S, dense) in sorted(R.aggregate("col", mat2).items()):
        total = sum(d.to_numpy().sum(axis=0) for d in dense) + (S if S is not None else 0.0)
        got += list(total)
    assert got == e["colSum_mat2"]
    col3 = R.project(mat2, 2, False, 3)
    assert [x for k in sorted(col3) for x in col3[k].tolist()] == e["project_col_3_mat2"]


def test_golden_test_sparse():
    g = json.load(open(os.path.join(GOLDEN, "test_sparse.json")))
    for name, full in (("spmat1", "S1_full"), ("spmat2", "S2_full")):
        d = g[name]
        a = np.asarray(g[full], dtype=np.float64)
        for s in (csc(d["numRows"], d["numCols"], d["colPtrs"], d["rowIndices"], d["values"]), as_csr(a)):
            assert np.array_equal(R.partial("row", s), a.sum(axis=1))
            assert np.array_equal(R.partial("col", s), a.sum(axis=0))
            assert R.partial("trace", s)[0] == np.trace(a)
            for i in range(3):
                assert np.array_equal(R.line_of(s, True, i), a[i, :])
                assert np.array_equal(R.line_of(s, False, i), a[:, i])
                for j in range(3):
                    assert R.entry_of(s, i, j) == a[i, j]


def int_dataset(rng, n, m, blk):
    """Integer-valued blocks without repeats: dense (both layouts), CSC and CSR, some absent, some empty."""
    ds = {}
    for i in range(-(-n // blk)):
        for j in range(-(-m // blk)):
            r, c = min(blk, n - i * blk), min(blk, m - j * blk)
            kind = rng.integers(0, 5)
            if kind == 4:
                continue
            a = rng.integers(-50, 50, (r, c)).astype(np.float64)
            a[rng.random((r, c)) < 0.7] = 0.0
            if kind == 0:
                ds[(i, j)] = O.DenseMatrix(r, c, np.ascontiguousarray(a.T).reshape(-1))
            elif kind == 1:
                ds[(i, j)] = O.DenseMatrix(r, c, np.ascontiguousarray(a).reshape(-1), True)
            elif kind == 2:
                ds[(i, j)] = O.DenseMatrix(r, c, np.ascontiguousarray(a.T).reshape(-1)).toSparse()
            else:
                ds[(i, j)] = as_csr(a)
    return ds


def test_against_the_oracle_on_integers():
    rng = np.random.default_rng(2)
    for n, m, blk in ((70, 50, 16), (64, 64, 16), (33, 33, 8)):
        ds = int_dataset(rng, n, m, blk)
        for op, fn in (("row", O.row_sum), ("col", O.col_sum)):
            want = fn(ds, n, m)
            got = R.aggregate(op, ds)
            assert sorted(got) == sorted(want)
            for key, (S, dense) in got.items():
                total = sum((d.to_numpy().sum(axis=1 if op == "row" else 0) for d in dense), np.zeros_like(want[key].values))
                assert np.array_equal(total + (S if S is not None else 0.0), want[key].values), (op, key)
        if n == m:
            (S, dense), = R.aggregate("trace", ds).values()
            total = sum(float(np.trace(d.to_numpy())) for d in dense) + (S[0] if S is not None else 0.0)
            assert total == O.trace(ds, n, m)[(0, 0)].values[0]
        for take_row in (True, False):
            for index in (0, blk - 1, blk, (n if take_row else m) - 1):
                want = O.project(ds, n, m, blk, take_row, index)
                got = R.project(ds, blk, take_row, index)
                assert sorted(got) == sorted(want)
                assert all(np.array_equal(got[k], want[k].values) for k in want)
        for i, j in ((0, 0), (n - 1, m - 1), (blk, blk - 1), (n // 2, m // 3)):
            want = O.selection(ds, n, m, blk, i, j)
            got = R.selection(ds, blk, i, j)
            assert sorted(got) == sorted(want) and all(got[k][0] == want[k].values[0] for k in want)


def test_repeats_order_and_signs():
    # three entries at (0, 0) in one CSC line: ((0 + 1e16) + 1) - 1e16 = 0 (1e16 + 1 rounds to 1e16); the last one is -1e16
    s = csc(2, 2, [0, 3, 3], [0, 0, 0], [1e16, 1.0, -1e16])
    assert R.partial("row", s).tolist() == [0.0, 0.0]
    assert R.partial("col", s).tolist() == [0.0, 0.0]
    assert R.partial("trace", s).tolist() == [0.0]
    assert R.entry_of(s, 0, 0) == -1e16 and R.line_of(s, True, 0).tolist() == [-1e16, 0.0]
    # the same entries stored in another order sum to 1: the order is part of the result
    assert R.partial("row", csc(2, 2, [0, 3, 3], [0, 0, 0], [1e16, -1e16, 1.0])).tolist() == [1.0, 0.0]
    # repeats across lines of a CSR block (row sums across rows of column 1): 0.1 + 0.2 in storage order, then the last wins
    t = csr(2, 2, [0, 1, 2], [1, 1], [0.1, 0.2])
    assert same(R.partial("col", t), [0.0, 0.1 + 0.2])
    assert same(R.line_of(t, False, 1), [0.1, 0.2])
    # -0.0: a sum starts at +0.0, so a stored -0.0 sums to +0.0; a slice keeps its sign
    z = csc(2, 2, [0, 1, 2], [1, 0], [-0.0, -0.0])
    assert same(R.partial("row", z), [0.0, 0.0]) and same(R.partial("col", z), [0.0, 0.0])
    assert same(R.line_of(z, True, 1), [-0.0, 0.0]) and same([R.entry_of(z, 0, 1)], [-0.0])
    # unsorted line with a repeat: the last stored entry of a position wins, every stored entry sums
    u = csc(4, 1, [0, 4], [3, 1, 3, 0], [1.0, 2.0, 5.0, 7.0])
    assert R.line_of(u, False, 0).tolist() == [7.0, 2.0, 0.0, 5.0]
    assert R.partial("row", u).tolist() == [7.0, 2.0, 0.0, 6.0] and R.partial("col", u).tolist() == [15.0]
    # non-finite values take part: Inf + -Inf is NaN; NaN spreads; a slice keeps them
    f = csr(2, 3, [0, 3, 4], [0, 2, 0, 1], [INF, NAN, -INF, 3.0])
    assert np.isnan(R.partial("row", f)[0]) and R.partial("row", f)[1] == 3.0
    assert np.isnan(R.partial("col", f)[0]) and R.partial("col", f)[1] == 3.0 and np.isnan(R.partial("col", f)[2])
    assert np.isnan(R.partial("trace", f)[0])  # (0, 0): Inf then -Inf
    assert same(R.line_of(f, True, 0), [-INF, 0.0, NAN])


def test_combine_in_ascending_block_index():
    # rowSum of one block row with three sparse blocks: S = ((0 + p0) + p1) + p2, in cid order
    a = csc(1, 1, [0, 1], [0], [1e16])
    b = csc(1, 1, [0, 1], [0], [1.0])
    c = csc(1, 1, [0, 1], [0], [-1e16])
    (S, dense), = R.aggregate("row", {(0, 2): c, (0, 0): a, (0, 1): b}).values()
    assert dense == [] and S.tolist() == [0.0]
    (S, _), = R.aggregate("row", {(0, 0): a, (0, 1): c, (0, 2): b}).values()
    assert S.tolist() == [1.0]
    # a line with a dense block lists it; its terms are every stored entry and dense element at the index
    d = O.DenseMatrix(1, 1, [2.0])
    (S, dense), = R.aggregate("col", {(0, 0): a, (1, 0): d}).values()
    assert S.tolist() == [1e16] and dense == [d]
    assert sorted(R.terms("col", {(0, 0): a, (1, 0): d}, (0, 0), 0).tolist()) == [2.0, 1e16]

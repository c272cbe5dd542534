"""GPU tests of dense x low-density sparse products computed from the stored entries of the sparse block (DESIGN section 4.5.2).

A dense-left x sparse-right pair takes the route when the right block holds at most kDspmmMaxDensity of its cells, its dims are
within the kernel's limits (rows and columns <= 1024, at least 128 columns; a left block with an even number of rows, 16 .. 1024)
and its output block has no pair on the dense engines; every other such pair is densified as before.  The route must give
A . toDense(S) up to rounding: the same ids, formats and flags, every k a term (sparse_sum_bound), the IEEE class of Inf * 0 for a
non-finite A(i, k) facing an implicit zero, and the last stored value of a repeated (k, j).

Every numeric case runs the three checks of test_gpu_spmm_edges.check and asserts its route through `dspmm_pairs` and the kernel
launch count."""
import os
import re

import numpy as np
import pytest

import matrel_b200 as mb
from matrel_b200.dataset import sprand
from oracle import matrel_oracle as O
from tests.exact_ref import ROOT, exact_dot, round_to_double
from tests.spmm_ref import segment_params, within
from tests.test_gpu_spmm_edges import LAYOUTS, check, csr_from_rows, dense, multiply, rand_csr, to_csc
from tests.test_gpu_streamed import _assert_identical, _dump, _streamed
from tests.test_gpu_unaligned import adopt_unaligned

pytestmark = pytest.mark.gpu

MAX_DIM = 1024
E_CAP = segment_params()["E_CAP"]
TAU = float(re.search(r"constexpr double kDspmmMaxDensity = ([0-9.e-]+);",
                      open(os.path.join(ROOT, "matrel_b200", "csrc", "abi_multiply.cpp")).read()).group(1))


@pytest.fixture(scope="module")
def sess():
    s = mb.MatfastSession(device=0, gemm_algo=1)
    yield s
    s.stop()


# ------------------------------------------------------------------------------------------------ operands
def rand_csc(rng, rows, cols, density, sort=True, dups=0.0):
    """Random CSC block (the CSR of its transpose, read as CSC): `dups` repeats an index in that share of columns."""
    t = rand_csr(rng, cols, rows, density, sort=sort, dups=dups)
    return O.SparseMatrix(rows, cols, t.colPtrs, t.rowIndices, t.values, False)


def sparse_blocks(rng, k, m, blk, density, fmt="csc", **kw):
    """k x m sparse operand; fmt 'csc', 'csr' or a function (kb, j) -> 'csc' / 'csr'."""
    out = {}
    for kb in range(-(-k // blk)):
        for j in range(-(-m // blk)):
            r, c = min(blk, k - kb * blk), min(blk, m - j * blk)
            f = fmt(kb, j) if callable(fmt) else fmt
            out[(kb, j)] = rand_csc(rng, r, c, density, **kw) if f == "csc" else rand_csr(rng, r, c, density, **kw)
    return out


def dense_blocks(M, blk, rowmajor=LAYOUTS["col"]):
    n, k = M.shape
    return {(i, kb): dense(M[i * blk:(i + 1) * blk, kb * blk:(kb + 1) * blk], rowmajor(i, kb))
            for i in range(-(-n // blk)) for kb in range(-(-k // blk))}


# ------------------------------------------------------------------------------------------------ the route, restated
def _is_gemm(a, b):
    if isinstance(a, O.DenseMatrix):
        return True
    return isinstance(b, O.SparseMatrix) and a.values.size / (a.numRows * a.numCols) > 0.1


def candidate(a, b):
    if not isinstance(a, O.DenseMatrix) or not isinstance(b, O.SparseMatrix):
        return False
    if not (0 < b.numRows <= MAX_DIM and 128 <= b.numCols <= MAX_DIM):
        return False
    if not (16 <= a.numRows <= MAX_DIM and a.numRows % 2 == 0):
        return False
    return b.values.size / (b.numRows * b.numCols) <= TAU


def plan(A, B):
    """{output block: [(a id, b id, routed)]} for the dense x sparse pairs of the product (join on k)."""
    outs = {}
    for (i, kb), a in A.items():
        for (kb2, j), b in B.items():
            if kb2 == kb:
                outs.setdefault((i, j), []).append(((i, kb), (kb2, j)))
    routes = {}
    for key, pairs in outs.items():
        other = any(_is_gemm(A[p[0]], B[p[1]]) and not candidate(A[p[0]], B[p[1]]) for p in pairs)
        routes[key] = [(pa, pb, candidate(A[pa], B[pb]) and not other) for pa, pb in pairs
                       if isinstance(A[pa], O.DenseMatrix) and isinstance(B[pb], O.SparseMatrix)]
    return routes


def expected(A, B, unaligned=False):
    """(routed pairs, kernel launches) of a product whose pairs are all dense x dense or dense x sparse, under gemm_algo 1.
    The route: 4 sptrans launches when a routed right block is CSR, the preparation, one EW_COPY when a routed left block is
    row-major or (`unaligned`) not 16-byte aligned, the flag pass, the kernel and the fix-up.  Densified right blocks: one launch
    each; the DMMA kernel: one."""
    pairs = [(pa, pb, ok) for r in plan(A, B).values() for pa, pb, ok in r]
    routed = [(pa, pb) for pa, pb, ok in pairs if ok]
    densified = {pb for pa, pb, ok in pairs if not ok}
    dd = any(isinstance(b, O.DenseMatrix) and any(kb == key[0] for (_, kb) in A) for key, b in B.items())
    launches = len(densified) + int(bool(densified) or dd)
    if routed:
        launches += 4 * any(B[pb].isTransposed for _, pb in routed) + (unaligned or any(A[pa].isTransposed for pa, _ in routed)) + 4
    return routed, launches


def run(s, A, B, n, k, m, blk, unaligned=False, **opts):
    """The product, with its route asserted: dspmm_pairs, dspmm_products and the launch count."""
    routed, launches = expected(A, B, unaligned)
    got, st = multiply(s, A, B, n, k, m, blk, **opts)
    assert st["dspmm_pairs"] == len(routed), (st["dspmm_pairs"], len(routed))
    assert st["dspmm_products"] == sum(B[pb].values.size * A[pa].numRows for pa, pb in routed)
    assert st["kernel_launches"] == launches, (st["kernel_launches"], launches)
    return got, st


def bits(blocks):
    return {key: m.values.view(np.int64).copy() for key, m in blocks.items()}


# ------------------------------------------------------------------------------------------------ shapes around every condition
SHAPES = [  # (A rows, k, S columns, blk): S columns 127 / 128 / 255 / 256 / 257 / 1024, A rows 14 .. 1024, k 127 / 128 / 129
    (64, 128, 128, 128),
    (64, 128, 127, 128),      # 127 columns: densified
    (16, 127, 255, 256),
    (14, 129, 256, 256),      # 14 rows: densified
    (17, 128, 257, 512),      # odd rows: densified
    (65, 128, 256, 256),      # odd rows: densified
    (1024, 1024, 1024, 1024),
    (600, 700, 1100, 512),    # ragged last blocks; the 76-column block column is densified
    (130, 129, 300, 256),     # ragged: 44-column block column densified, the rest routed
]


@pytest.mark.parametrize("n,k,m,blk", SHAPES)
def test_shapes(sess, n, k, m, blk):
    rng = np.random.default_rng(n * 7 + k * 3 + m)
    A = dense_blocks(rng.uniform(-1, 1, (n, k)), blk)
    B = sparse_blocks(rng, k, m, blk, 0.01)
    got, _ = run(sess, A, B, n, k, m, blk)
    check(got, A, B, n, k, m, blk, rng)


@pytest.mark.parametrize("fmt", ["csc", "csr", "mixed"])
@pytest.mark.parametrize("layout", ["col", "row", "mixed"])
@pytest.mark.parametrize("sort", [True, False])
def test_formats_and_layouts(sess, fmt, layout, sort):
    rng = np.random.default_rng(["csc", "csr", "mixed"].index(fmt) * 10 + ["col", "row", "mixed"].index(layout) * 2 + sort)
    n, k, m, blk = 300, 512, 512, 256
    A = dense_blocks(rng.uniform(-1, 1, (n, k)), blk, LAYOUTS[layout])
    f = (lambda kb, j: "csr" if (kb + j) % 2 else "csc") if fmt == "mixed" else fmt
    B = sparse_blocks(rng, k, m, blk, 0.01, f, sort=sort)
    got, _ = run(sess, A, B, n, k, m, blk)
    check(got, A, B, n, k, m, blk, rng)


@pytest.mark.parametrize("fmt", ["csc", "csr"])
def test_empty_columns_empty_and_absent_blocks(sess, fmt):
    rng = np.random.default_rng(5)
    n, k, m, blk = 256, 768, 768, 256
    A = dense_blocks(rng.uniform(-1, 1, (n, k)), blk)
    del A[(0, 2)]                                                    # absent left block
    B = sparse_blocks(rng, k, m, blk, 0.003, fmt)                    # most columns empty
    B[(1, 1)] = csr_from_rows(256, 256, [[] for _ in range(256)], rng) if fmt == "csr" else \
        to_csc(csr_from_rows(256, 256, [[] for _ in range(256)], rng))   # no stored entry
    del B[(0, 2)]                                                    # absent right block
    got, _ = run(sess, A, B, n, k, m, blk)
    check(got, A, B, n, k, m, blk, rng)


@pytest.mark.parametrize("place", ["spread", "one_segment"])
@pytest.mark.parametrize("side", [-1, 1])
def test_density_around_tau(sess, side, place):
    """nnz = tau * cells - 1 (routed) and + 1 (densified).  "one_segment" puts every entry into the first 128 rows of the first
    256 columns: that (strip, chunk) segment holds more than E_CAP entries, so the kernel reads it through the global-memory
    window, next to empty segments."""
    rng = np.random.default_rng(11)
    n, k, m, blk = 256, 256, 512, 512
    A = dense_blocks(rng.uniform(-1, 1, (n, k)), blk)
    nnz = int(TAU * k * m) + side
    M = np.zeros((k, m))
    region = M if place == "spread" else M[:128, :256]
    flat = rng.choice(region.size, nnz, replace=False)
    np.put(region, flat, rng.uniform(-1, 1, nnz))
    B = {(0, 0): O.DenseMatrix(k, m, np.ascontiguousarray(M.T).reshape(-1)).toSparse()}
    assert B[(0, 0)].values.size == nnz
    if place == "one_segment":
        assert nnz > E_CAP
    got, st = run(sess, A, B, n, k, m, blk)
    assert (st["dspmm_pairs"] > 0) == (side < 0)
    check(got, A, B, n, k, m, blk, rng)


# ------------------------------------------------------------------------------------------------ mixed output blocks
def test_dense_pair_next_to_dense_sparse_is_densified(sess):
    """A dense x dense pair in the block keeps every pair of it on the dense engine: under gemm_algo 0 the product runs on the
    same engine as with B's blocks stored dense."""
    rng = np.random.default_rng(21)
    n, k, m, blk = 2048, 2048, 2048, 1024
    A = dense_blocks(rng.uniform(-1, 1, (n, k)), blk)
    B = {(0, 0): dense(rng.uniform(-1, 1, (blk, blk)), False), (1, 0): rand_csc(rng, blk, blk, 0.01),
         (0, 1): rand_csr(rng, blk, blk, 0.01), (1, 1): dense(rng.uniform(-1, 1, (blk, blk)), True)}
    got, st = run(sess, A, B, n, k, m, blk)
    assert st["dspmm_pairs"] == 0
    check(got, A, B, n, k, m, blk, rng, samples=40)
    Bd = {key: dense(b.to_numpy(), False) for key, b in B.items()}
    for algo in (0, 1):
        _, st_sp = multiply(sess, A, B, n, k, m, blk, gemm_algo=algo)
        _, st_d = multiply(sess, A, Bd, n, k, m, blk, gemm_algo=algo)
        assert st_sp["tc_gemm_launches"] == st_d["tc_gemm_launches"] == (algo == 0), algo
        assert st_sp["dspmm_pairs"] == 0


def test_sparse_dense_next_to_dense_sparse_accumulates(sess):
    """Block (0, 0) = CSR(0, 0) x dense(0, 0) (pipelined sparse x dense kernel) + dense(0, 1) x CSC(1, 0) (the route, on top)."""
    rng = np.random.default_rng(22)
    n, k, m, blk = 256, 512, 256, 256
    A = {(0, 0): rand_csr(rng, 256, 256, 0.05), (0, 1): dense(rng.uniform(-1, 1, (256, 256)), False)}
    B = {(0, 0): dense(rng.uniform(-1, 1, (256, 256)), False), (1, 0): rand_csc(rng, 256, 256, 0.01)}
    got, st = multiply(sess, A, B, n, k, m, blk)
    assert st["dspmm_pairs"] == 1
    assert st["kernel_launches"] == 3 + 4    # sparse x dense: prep, B transpose, kernel; the route: prep, flags, kernel, fix-up
    check(got, A, B, n, k, m, blk, rng)


def test_sparse_sparse_next_to_dense_sparse_is_dense(sess):
    """A low-density sparse x sparse pair next to a routed pair: the block ends dense, as LocalMatrix.add makes it."""
    rng = np.random.default_rng(23)
    n, k, m, blk = 256, 512, 256, 256
    A = {(0, 0): rand_csc(rng, 256, 256, 0.01), (0, 1): dense(rng.uniform(-1, 1, (256, 256)), True)}
    B = {(0, 0): rand_csc(rng, 256, 256, 0.01), (1, 0): rand_csr(rng, 256, 256, 0.01)}
    got, st = multiply(sess, A, B, n, k, m, blk)
    assert st["dspmm_pairs"] == 1 and st["spgemm_pairs"] == 0
    # B(0, 0) densified and the per-pair CSC x dense kernel; the route: sptrans (B(1, 0) is CSR), preparation, EW_COPY (A(0, 1)
    # is row-major), flags, kernel, fix-up
    assert st["kernel_launches"] == 1 + 1 + 4 + 1 + 1 + 3, st["kernel_launches"]
    assert isinstance(got[(0, 0)], mb.DenseMatrix)
    check(got, A, B, n, k, m, blk, rng)


@pytest.mark.parametrize("layout", ["col", "mixed"])
def test_unaligned_left_blocks_take_the_scratch_copy(sess, layout):
    """Left blocks adopted at an odd element offset (8- but not 16-byte aligned) go through the EW_COPY into the scratch like
    row-major ones, so the route does not depend on addresses."""
    rng = np.random.default_rng(81 + len(layout))
    n, k, m, blk = 512, 512, 512, 256
    A = dense_blocks(rng.uniform(-1, 1, (n, k)), blk, LAYOUTS[layout])
    B = sparse_blocks(rng, k, m, blk, 0.01)
    dA, keep = adopt_unaligned(sess, A)
    got, _ = run(sess, A, B, n, k, m, blk, unaligned=True, dA=dA)
    check(got, A, B, n, k, m, blk, rng)
    del dA, keep


def test_more_than_65535_left_blocks():
    """65537 routed left blocks of 128 rows against one 128 x 128 CSC block: the flag pass has one CTA column per left block,
    past the 65535 limit of a grid's y and z dimensions.  An Inf in the last block must still reach C."""
    nb, blk = 65537, 128
    R = nb * blk
    rng = np.random.default_rng(91)
    with mb.MatfastSession(device=0, gemm_algo=1) as s:
        A = s.rand(R, blk, blk, 5)
        S = sprand(s, blk, blk, blk, 0.01, 6, csr=False)
        last = rng.uniform(-1, 1, (blk, blk))
        last[3, 5] = np.inf
        A.put_block(nb - 1, 0, mb.DenseMatrix.from_numpy(last))
        s.sync()
        s.reset_stats()
        C = A.matrixMultiply(R, blk, S, blk, blk, blk)
        s.sync()
        st = s.stats()
        assert st["dspmm_pairs"] == nb
        assert st["kernel_launches"] == 4, st["kernel_launches"]   # preparation, flags, kernel, fix-up
        Sd = S.get_block(0, 0).to_numpy()
        for i in (0, 1, 65534, 65535, nb - 1) + tuple(int(x) for x in rng.integers(nb, size=3)):
            a = last if i == nb - 1 else A.get_block(i, 0).to_numpy()
            got = C.get_block(i, 0).to_numpy()
            with np.errstate(invalid="ignore"):
                want = a @ Sd
            assert np.array_equal(np.isnan(got), np.isnan(want)), i
            fin = np.isfinite(want)
            bound = 1.01 * (blk + 2) * 2.0 ** -53 * (np.abs(np.where(np.isfinite(a), a, 0)) @ np.abs(Sd)) + 2.0 ** -1060
            assert (np.abs(got - want)[fin] <= bound[fin]).all(), i
        assert np.isnan(C.get_block(nb - 1, 0).to_numpy()[3]).sum() == int((Sd[5] == 0).sum())


# ------------------------------------------------------------------------------------------------ values
def test_nonfinite_left_values(sess):
    """+-Inf and NaN in A against implicit zeros, stored zeros and stored values of S, in rows with and without stored partners.
    Rows of A without a non-finite value are bit for bit those of the all-finite run."""
    rng = np.random.default_rng(31)
    n, k, m, blk = 256, 512, 512, 256
    M = rng.uniform(-1, 1, (n, k))
    B = sparse_blocks(rng, k, m, blk, 0.005)
    # row 5 of S's first k-block stores a zero in every column of block column 0; row 300 (k-block 1) stores nothing
    b = B[(0, 0)].to_numpy()
    b[5, :] = 0.0
    b[7, :] = 1.5          # stored in every column
    rows = [np.flatnonzero(b[:, c]).tolist() for c in range(b.shape[1])]
    rows = [sorted(set(r) | {5, 7}) for r in rows]
    B[(0, 0)] = _csc_of(b, rows)
    b1 = B[(1, 0)].to_numpy()
    b1[300 - 256, :] = 0.0
    B[(1, 0)] = O.DenseMatrix(*b1.shape, np.ascontiguousarray(b1.T).reshape(-1)).toSparse()
    bad = M.copy()
    bad[3, 5] = np.inf        # stored zeros: NaN everywhere in block column 0; mostly implicit zeros in block column 1
    bad[10, 7] = -np.inf      # stored 1.5 in block column 0: -Inf there; mostly implicit zeros in block column 1: NaN
    bad[20, 300] = np.nan     # nothing stored in row 300: NaN through implicit zeros
    bad[30, 40] = np.inf      # a row with an ordinary k
    bad[40, 7] = np.nan
    nf_rows = {3, 10, 20, 30, 40}
    A_bad, A_ok = dense_blocks(bad, blk), dense_blocks(M, blk)
    got, _ = run(sess, A_bad, B, n, k, m, blk)
    ok, _ = run(sess, A_ok, B, n, k, m, blk)
    G = check(got, A_bad, B, n, k, m, blk, rng)
    G0 = O.assemble(ok, n, m, blk)
    keep = [i for i in range(n) if i not in nf_rows]
    assert np.array_equal(G[keep].view(np.int64), G0[keep].view(np.int64))
    assert np.isnan(G[3, :256]).all() and np.isnan(G[20]).all() and np.isnan(G[40]).all()
    assert (G[10, :256] == -np.inf).all() and np.isnan(G[10, 256:]).any() and np.isnan(G[30]).any()


def _csc_of(b, rows_per_col):
    """CSC block storing exactly rows_per_col[c] of column c (zeros included) with the values of b."""
    ptr = np.cumsum([0] + [len(r) for r in rows_per_col]).astype(np.int32)
    idx = np.concatenate([np.asarray(r, dtype=np.int32) for r in rows_per_col])
    val = np.concatenate([b[r, c] for c, r in enumerate(rows_per_col)]).astype(np.float64)
    return O.SparseMatrix(b.shape[0], b.shape[1], ptr, idx, val, False)


@pytest.mark.parametrize("fmt", ["csc", "csr"])
@pytest.mark.parametrize("sort", [True, False])
def test_repeated_coordinates_keep_the_last_value(sess, fmt, sort):
    rng = np.random.default_rng(41)
    n, k, m, blk = 128, 256, 256, 256
    A = dense_blocks(rng.uniform(-1, 1, (n, k)), blk)
    B = sparse_blocks(rng, k, m, blk, 0.01, fmt, sort=sort, dups=0.5)
    b = B[(0, 0)]
    assert np.diff(b.colPtrs).sum() > np.count_nonzero(b.to_numpy())            # some coordinates repeat
    got, _ = run(sess, A, B, n, k, m, blk)
    G = check(got, A, B, n, k, m, blk, rng)
    last = O.assemble(A, n, k, blk) @ b.to_numpy()                               # toArray: the last stored value
    assert np.allclose(G, last, rtol=0, atol=1e-12)


def test_deterministic_and_the_same_under_every_gemm_algo(sess):
    rng = np.random.default_rng(51)
    n, k, m, blk = 1024, 2048, 2048, 1024
    A = dense_blocks(rng.uniform(-1, 1, (n, k)), blk, LAYOUTS["mixed"])
    B = sparse_blocks(rng, k, m, blk, 0.005, lambda kb, j: "csr" if j else "csc")
    first, _ = run(sess, A, B, n, k, m, blk)
    again, _ = run(sess, A, B, n, k, m, blk)
    want = bits(first)
    assert bits(again).keys() == want.keys() and all(np.array_equal(bits(again)[key], want[key]) for key in want)
    for algo in (0, 3):
        got, st = run(sess, A, B, n, k, m, blk, gemm_algo=algo)
        assert st["dspmm_pairs"] == 4
        g = bits(got)
        assert all(np.array_equal(g[key], want[key]) for key in want), algo
    check(first, A, B, n, k, m, blk, rng, samples=60)


# ------------------------------------------------------------------------------------------------ streamed
@pytest.mark.parametrize("mixed", [False, True], ids=["colmajor_csc", "mixed"])
@pytest.mark.parametrize("residence", ["A", "B", "AB"])
def test_streamed_matches_resident(residence, mixed):
    """Every tile routes its pairs: 4 launches per tile with column-major A and CSC B (preparation, flags, kernel, fix-up), up to
    4 + 4 (sptrans) + 1 (EW_COPY) when a tile holds CSR or row-major blocks."""
    rng = np.random.default_rng(61)
    M, K, N, blk = 1024, 768, 1024, 256
    Ab = {key: mb.DenseMatrix.from_numpy(rng.uniform(-1, 1, (256, 256)), transposed_storage=mixed and (key[0] + key[1]) % 2 == 1)
          for key in [(i, kb) for i in range(4) for kb in range(3)]}
    Bo = sparse_blocks(rng, K, N, blk, 0.01, lambda kb, j: "csr" if mixed and (kb + j) % 2 else "csc")
    Bb = {key: mb.SparseMatrix(b.numRows, b.numCols, b.colPtrs, b.rowIndices, b.values, b.isTransposed) for key, b in Bo.items()}

    def load(s, blocks, host):
        rows = [mb.MatrixBlock(i, j, x) for (i, j), x in sorted(blocks.items())]
        return s.createHostDataset(rows) if host else s.createDataset(rows)
    with mb.MatfastSession(device=0) as s:
        s.reset_stats()
        want = _dump(load(s, Ab, False).matrixMultiply(M, K, load(s, Bb, False), K, N, blk))
        assert s.stats()["dspmm_pairs"] == 4 * 3 * 4
        C, st = _streamed(s, load(s, Ab, "A" in residence), load(s, Bb, "B" in residence), M, K, N, blk)
        t = st["stream_tiles"]
        assert C.isHost and t >= 2, t
        assert st["dspmm_pairs"] == 4 * 3 * 4
        if mixed:
            assert 4 * t < st["kernel_launches"] <= 9 * t, (st["kernel_launches"], t)
        else:
            assert st["kernel_launches"] == 4 * t, (st["kernel_launches"], t)
        _assert_identical(_dump(C), want)


# ------------------------------------------------------------------------------------------------ the capability
def test_capability_wt_v_n131072():
    """W^T V with W a 131072 x 1024 rand dataset and V sprand 131072^2 at 1e-4 (CSC), blk 1024: the dense images of V's blocks
    alone would take 128 GiB.  Freivalds: C x against W^T (V x), V x on the sparse x dense kernel; exact entries at samples."""
    N, r, blk, d = 131072, 1024, 1024, 1e-4
    nb = N // blk
    with mb.MatfastSession(device=0) as s:
        W = s.rand(N, r, blk, 3)
        V = sprand(s, N, N, blk, d, 4, csr=False)
        Wt = W.transpose()
        s.sync()
        s.reset_stats()
        C = Wt.matrixMultiply(r, N, V, N, N, blk)
        s.sync()
        st = s.stats()
        assert st["dspmm_pairs"] == nb * nb
        assert st["kernel_launches"] == 5   # preparation, EW_COPY of the row-major W^T blocks, flags, kernel, fix-up
        rng = np.random.default_rng(71)
        x = rng.uniform(-1, 1, N)
        X = s.createDataset(mb.MatrixBlock(kb, 0, mb.DenseMatrix.from_numpy(x[kb * blk:(kb + 1) * blk, None])) for kb in range(nb))
        Cx = C.matrixMultiply(r, N, X, N, 1, blk).toNumpy(r, 1, blk)[:, 0]
        Vx = V.matrixMultiply(N, N, X, N, 1, blk)
        WtVx = Wt.matrixMultiply(r, N, Vx, N, 1, blk).toNumpy(r, 1, blk)[:, 0]
        scale = float(np.abs(WtVx).max())
        assert np.abs(Cx - WtVx).max() <= 1e-10 * scale, float(np.abs(Cx - WtVx).max() / scale)
        # exact entries: C[i, c] = sum over the stored (k, c) of V of W[k, i] V[k, c]
        for cb in (0, 77, nb - 1):
            vb = {kb: V.get_block(kb, cb) for kb in range(nb)}
            cblk = C.get_block(0, cb).to_numpy()
            cols = rng.choice(blk, 4, replace=False).tolist() + [0, blk - 1]
            need = {kb for kb in range(nb) for c in cols if vb[kb].colPtrs[c + 1] > vb[kb].colPtrs[c]}
            wb = {kb: W.get_block(kb, 0).to_numpy() for kb in need}
            for c in cols:
                ks, vs = [], []
                for kb in range(nb):
                    lo, hi = vb[kb].colPtrs[c], vb[kb].colPtrs[c + 1]
                    ks += [(kb, int(t)) for t in vb[kb].rowIndices[lo:hi]]
                    vs += vb[kb].values[lo:hi].tolist()
                for i in rng.choice(r, 6, replace=False).tolist() + [0, r - 1]:
                    a = np.array([wb[kb][t, i] for kb, t in ks])
                    exact = exact_dot(a, np.array(vs))
                    bound = 1.01 * (len(vs) + 2) * 2.0 ** -53 * float(np.abs(a * np.array(vs)).sum()) + (len(vs) + 4) * 2.0 ** -1074
                    assert within(cblk[i, c], exact, bound), (cb, c, i, float(cblk[i, c]), float(round_to_double(exact)))

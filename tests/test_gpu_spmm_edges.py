"""GPU tests of the sparse x dense multiply on every kernel route, at the shapes, segment sizes, layouts and values where the
kernels branch, against the exact sparse reference of tests/spmm_ref.py.

The host picks a route per output block (abi_multiply.cpp): the pipelined TMA kernel (spmm2_prep_kernel + spmm2_kernel, plus an
EW_COPY transpose of column-major B) for CSR blocks of at most 1024 x 1024 when m >= 128, n >= 16, n even and every B base is
16-byte aligned; the fused shared-memory kernel (spmm_fused_kernel) for the other CSR blocks of that size; one spmm_csr_kernel
launch per pair above 1024; one spmm_csc_kernel launch per CSC pair.  Every case asserts its route through the launch count.

Every numeric case gets three checks (check):
  (a) ids, presence, formats and flags equal the oracle's;
  (b) the WHOLE product against scipy.sparse (stored entries only, like BLAS.gemmsdd) within sparse_sum_bound for the kernel
      plus the same bound for scipy's own order, non-finite positions exactly equal;
  (c) exact entries within sparse_sum_bound alone at sampled positions and next to every strip, column tile, chunk, block and
      matrix edge; non-finite entries must have the IEEE outcome of their terms."""
import numpy as np
import pytest

import matrel_b200 as mb
from matrel_b200 import _native as N
from oracle import matrel_oracle as O
from tests.exact_ref import alpha_of, exact_entries, fp64_dot_bound, moduli_for, oz2_bound, round_to_double
from tests.spmm_ref import (classify, exact_sparse_entries, nonfinite_class, reference_product, segment_params,
                            sparse_sum_bound, within)
from tests.util import REL_TOL, assert_same_dataset, from_dataset, to_dataset

pytestmark = pytest.mark.gpu

SEG = segment_params()
TM, TN, KC, E_CAP = SEG["TM"], SEG["TN"], SEG["KC"], SEG["E_CAP"]
MAX_DIM = 1024                                  # kSpmmMaxDim: m and kdim limit of the fused and pipelined kernels
DEFAULTS = {"gemm_algo": 1, "spmm_algo": 0, "gemm_variant": -1}


@pytest.fixture(scope="module")
def sess():
    s = mb.MatfastSession(device=0, gemm_algo=1)
    yield s
    s.stop()


# ------------------------------------------------------------------------------------------------ operands
def csr_from_rows(rows, cols, row_cols, rng, values=None):
    """CSR block whose row r stores the columns row_cols[r] in the given order, with U(-1, 1) values (or values[r])."""
    ptr = np.cumsum([0] + [len(c) for c in row_cols]).astype(np.int32)
    idx = np.concatenate([np.asarray(c, dtype=np.int32) for c in row_cols]) if ptr[-1] else np.zeros(0, np.int32)
    val = np.concatenate([np.asarray(v, dtype=np.float64) for v in values]) if values is not None else rng.uniform(-1, 1, idx.size)
    assert len(row_cols) == rows and val.size == idx.size
    return O.SparseMatrix(rows, cols, ptr, idx, val, True)


def rand_csr(rng, rows, cols, density, sort=True, dups=0.0):
    """Random CSR block; `dups`: share of rows that repeat one of their column indices."""
    row_cols = []
    for _ in range(rows):
        c = np.flatnonzero(rng.random(cols) < density)
        if c.size and rng.random() < dups:
            c = np.append(c, c[rng.integers(c.size)])
        if not sort:
            rng.shuffle(c)
        row_cols.append(c)
    return csr_from_rows(rows, cols, row_cols, rng)


def to_csc(a):
    """The same stored entries (duplicates and zeros included) as a CSC block."""
    major = np.repeat(np.arange(a.numRows), np.diff(a.colPtrs))
    order = np.lexsort((major, a.rowIndices))                 # by column, rows ascending
    ptr = np.concatenate([[0], np.cumsum(np.bincount(a.rowIndices, minlength=a.numCols))]).astype(np.int32)
    return O.SparseMatrix(a.numRows, a.numCols, ptr, major[order].astype(np.int32), a.values[order], False)


def dense(a, rowmajor):
    a = np.asarray(a, dtype=np.float64)
    if rowmajor:
        return O.DenseMatrix(a.shape[0], a.shape[1], np.ascontiguousarray(a).reshape(-1), True)
    return O.DenseMatrix(a.shape[0], a.shape[1], np.ascontiguousarray(a.T).reshape(-1), False)


def blocks_of(M, blk, rowmajor=lambda i, j: False):
    n, m = M.shape
    return {(i, j): dense(M[i * blk:(i + 1) * blk, j * blk:(j + 1) * blk], rowmajor(i, j))
            for i in range(-(-n // blk)) for j in range(-(-m // blk))}


LAYOUTS = {"col": lambda i, j: False, "row": lambda i, j: True, "mixed": lambda i, j: (i + j) % 2 == 1}


def sparse_rows(rng, n, k, blk, density, **kw):
    return {(i, kb): rand_csr(rng, min(blk, n - i * blk), min(blk, k - kb * blk), density, **kw)
            for i in range(-(-n // blk)) for kb in range(-(-k // blk))}


# ------------------------------------------------------------------------------------------------ routes
def table_route(m, n, spmm_algo=0, aligned=True):
    """The host's choice for the CSR pairs (m, kdim <= 1024) of an m x n output block."""
    return "pipelined" if spmm_algo != 1 and m >= 128 and n >= 16 and n % 2 == 0 and aligned else "fused"


def plan_routes(A, B, spmm_algo=0, aligned=True):
    """(expected kernel launches, set of routes used) of the multiply.  Per-pair pairs cost one launch each, the fused and the
    pipelined kernels one launch for all their output blocks (+ preparation + one transpose of the column-major B blocks),
    densified sparse B blocks one launch each and dense x dense pairs one DMMA launch."""
    perpair, routes, colmajor, gemm, densified = 0, set(), False, False, set()
    for (i, kb), a in A.items():
        for (kb2, j), b in B.items():
            if kb2 != kb:
                continue
            if isinstance(a, O.DenseMatrix):
                gemm = True
                continue
            if isinstance(b, O.SparseMatrix):
                assert b.values.size / (b.numRows * b.numCols) > 0.1
                densified.add((kb2, j))
            if not a.isTransposed:
                perpair += 1
                routes.add("csc")
            elif a.numRows > MAX_DIM or a.numCols > MAX_DIM:
                perpair += 1
                routes.add("csr")
            else:
                r = table_route(a.numRows, b.numCols, spmm_algo, aligned)
                routes.add(r)
                colmajor |= r == "pipelined" and (isinstance(b, O.SparseMatrix) or not b.isTransposed)
    launches = perpair + len(densified) + gemm + ("fused" in routes) + ("pipelined" in routes) * (2 + colmajor)
    return launches, routes


def multiply(s, A, B, n, k, m, blk, dA=None, dB=None, **opts):
    """The product as a block dict plus the statistics of the multiply call alone; options are restored afterwards."""
    dA = dA if dA is not None else to_dataset(s, A)
    dB = dB if dB is not None else to_dataset(s, B)
    s.sync()
    for key, v in {**DEFAULTS, **opts}.items():
        s.set_option(key, v)
    try:
        s.reset_stats()
        ds = dA.matrixMultiply(n, k, dB, k, m, blk)
        st = s.stats()
        return from_dataset(ds), st
    finally:
        for key, v in DEFAULTS.items():
            s.set_option(key, v)


def run_route(s, A, B, n, k, m, blk, route, aligned=True, **kw):
    """Multiply and assert that `route` served the sparse pairs, with the launch count as the witness."""
    launches, routes = plan_routes(A, B, kw.get("spmm_algo", 0), aligned)
    assert route in routes, (route, routes)
    got, st = multiply(s, A, B, n, k, m, blk, **kw)
    assert st["kernel_launches"] == launches, (route, routes, st["kernel_launches"], launches)
    return got


# ------------------------------------------------------------------------------------------------ checks
def edge_indices(N, blk, steps):
    idx = {0, N - 1}
    for b0 in range(0, N, blk):
        hi = min(N, b0 + blk)
        for step in steps:
            for x in range(b0, hi + 1, step):
                idx.update((x - 1, x))
        idx.update((b0 - 1, b0, hi - 1))
    return sorted(i for i in idx if 0 <= i < N)


def positions(rng, n, m, blk, samples=200, cap=400):
    rows, cols = edge_indices(n, blk, (TM, KC, 16)), edge_indices(m, blk, (TN, KC))
    grid = [(i, j) for i in rows for j in cols]
    if len(grid) > cap:
        grid = [grid[t] for t in rng.choice(len(grid), cap, replace=False)]
    pos = set(grid) | {(n - 1, m - 1), (0, 0), (n - 1, 0), (0, m - 1)}
    pos |= {(i, int(rng.integers(m))) for i in rows} | {(int(rng.integers(n)), j) for j in cols}
    pos |= {(int(rng.integers(n)), int(rng.integers(m))) for _ in range(samples)}
    return sorted(pos)


def check(got, A, B, n, k, m, blk, rng, samples=200, rows=None):
    """(a), (b) and (c) above; `rows`: restrict (b) and (c) to these output rows (the others are checked by the caller)."""
    G = O.assemble(got, n, m, blk)
    ref = reference_product(A, B, n, k, m, blk)
    S = sparse_sum_bound(A, B, n, k, m, blk)
    sel = np.zeros(n, dtype=bool)
    sel[rows if rows is not None else slice(None)] = True
    fin = np.isfinite(ref)
    with np.errstate(invalid="ignore"):                                                              # (b)
        nf = ~fin & sel[:, None] & ~((G == ref) | (np.isnan(G) & np.isnan(ref)))
        assert not nf.any(), ("non-finite entries", [(int(i), int(j), float(G[i, j]), float(ref[i, j])) for i, j in np.argwhere(nf)[:8]])
        bad = fin & ~(np.abs(G - ref) <= 2 * S) & sel[:, None]
    assert not bad.any(), ("whole product", np.argwhere(bad)[:5].tolist())
    pos = [(i, j) for i, j in positions(rng, n, m, blk, samples) if sel[i]]                           # (c)
    classes = nonfinite_class(A, B, n, k, m, blk, pos)
    for (i, j), c in zip(pos, classes):
        assert classify(G[i, j]) == c, ("IEEE class", i, j, float(G[i, j]), c)
    fpos = [p for p, c in zip(pos, classes) if c == "finite"]
    for (i, j), x in zip(fpos, exact_sparse_entries(A, B, n, k, m, blk, fpos)):
        want = round_to_double(x)
        assert (G[i, j] == want) if not np.isfinite(want) else within(G[i, j], x, S[i, j]), \
            ("exact entry", i, j, float(G[i, j]), want, float(S[i, j]))
    assert_same_dataset(got, O.matrix_multiply(A, n, k, B, k, m, blk), tol=REL_TOL)                   # (a)
    return G


def same_bits(x, y):
    assert sorted(x) == sorted(y)
    for key in x:
        assert np.array_equal(x[key].values, y[key].values, equal_nan=True), key


# ------------------------------------------------------------------------------------------------ shapes around every threshold
# One block row with four k-blocks (the last one kdim = klast), so the output block has four sparse pairs of two kdims.
SHAPES = [  # rows (m), cols (n), klast, B layout
    (127, 64, 1, "col"), (128, 16, 127, "row"), (129, 14, 128, "mixed"), (255, 15, 129, "col"), (256, 17, 388, "row"),
    (257, 18, 1024, "mixed"), (1000, 65, 388, "col"), (1024, 66, 129, "row"), (1000, 130, 1, "mixed"), (1024, 1, 127, "col"),
    (256, 64, 128, "col"), (129, 130, 1024, "row"),
]


@pytest.mark.parametrize("rows,cols,klast,layout", SHAPES, ids=[f"{a}x{b}-k{c}-{d}" for a, b, c, d in SHAPES])
def test_shapes_around_every_threshold(sess, rows, cols, klast, layout):
    rng = np.random.default_rng(rows * 1000 + cols + klast)
    blk = MAX_DIM
    k = 3 * blk + klast
    A = sparse_rows(rng, rows, k, blk, 0.03)
    B = blocks_of(rng.uniform(-1, 1, (k, cols)), blk, LAYOUTS[layout])
    route = table_route(rows, cols)
    got = run_route(sess, A, B, rows, k, cols, blk, route)
    check(got, A, B, rows, k, cols, blk, rng)


@pytest.mark.parametrize("n,k,m,blk,routes", [
    (700, 3 * 256 + 100, 300, 256, {"pipelined"}),            # ragged strips (188 rows), chunks (100) and column tiles (44)
    (600, 4 * 256, 270, 256, {"pipelined", "fused"}),         # last block row of 88 rows takes the fused kernel, the rest pipelined
    (2048 + 300, 2 * 2048 + 300, 96, 2048, {"csr", "pipelined"}),  # blk 2048: per-pair CSR; the 300 x 300 corner pair pipelined
    (2048, 3 * 2048, 40, 2048, {"csr"}),
])
def test_multi_block_products_and_blk_2048(sess, n, k, m, blk, routes):
    rng = np.random.default_rng(n + k + m)
    A = sparse_rows(rng, n, k, blk, 0.02)
    B = blocks_of(rng.uniform(-1, 1, (k, m)), blk, LAYOUTS["mixed"])
    launches, used = plan_routes(A, B)
    assert used == routes
    got, st = multiply(sess, A, B, n, k, m, blk)
    assert st["kernel_launches"] == launches
    check(got, A, B, n, k, m, blk, rng)
    if "csr" in routes:                                       # per-pair CSR is deterministic
        again, _ = multiply(sess, A, B, n, k, m, blk)
        same_bits(got, again)


# ------------------------------------------------------------------------------------------------ segment capacity
def capacity_operands(rng):
    """Block row of 500 rows (strips of 256 and a ragged 244) x four k-blocks of 512 (chunks of 128), 200 columns.
    Block (0, 0), strip 0:
      chunk 0: rows 0-4 hold all 128 columns, row 5 holds 24          -> exactly E_CAP entries (shared memory)
      chunk 1: rows 0-4 full, row 5 holds 25                          -> E_CAP + 1 (global memory, 32-entry window)
      chunk 2: rows 16-18 hold 31 / 32 / 33 entries, rows 32-37 full  -> global; the window refills mid-row and across rows;
               warps 0, 3-15 own no entry of the chunk
      chunk 3: a few entries                                          -> shared: one tile mixes shared and global chunks
    Strip 1 (rows 256-499): chunk 0 dense enough for the global path with short rows, chunk 1 empty.
    Block (0, 2) has nnz = 0; blocks (0, 1) and (0, 3) are random."""
    assert E_CAP - 5 * KC > 0 and 5 * KC + 33 > E_CAP
    blk, rows, kdim = 512, 500, 512
    row_cols = [[] for _ in range(rows)]
    for r in range(5):
        row_cols[r] += list(range(0, KC)) + list(range(KC, 2 * KC))
    row_cols[5] += list(rng.choice(KC, E_CAP - 5 * KC, replace=False)) + list(KC + rng.choice(KC, E_CAP - 5 * KC + 1, replace=False))
    for r, ln in zip((16, 17, 18), (31, 32, 33)):
        row_cols[r] += list(2 * KC + rng.choice(KC, ln, replace=False))
    for r in range(32, 38):
        row_cols[r] += list(range(2 * KC, 3 * KC))
    for r in rng.choice(np.arange(40, 256), 20, replace=False):
        row_cols[r] += [3 * KC + int(rng.integers(kdim - 3 * KC))]
    for r in range(256, rows):
        row_cols[r] += list(np.flatnonzero(rng.random(KC) < 0.08)) + list(2 * KC + np.flatnonzero(rng.random(2 * KC) < 0.01))
    row_cols = [sorted(set(c)) for c in row_cols]
    a00 = csr_from_rows(rows, kdim, row_cols, rng)
    ptr = a00.colPtrs
    seg = [sum(1 for c in row_cols[r] if q * KC <= c < (q + 1) * KC) for q in range(4) for r in range(TM)]
    per_chunk = [sum(seg[q * TM:(q + 1) * TM]) for q in range(4)]
    assert per_chunk[0] == E_CAP and per_chunk[1] == E_CAP + 1 and per_chunk[2] > E_CAP and per_chunk[3] <= E_CAP
    assert int(ptr[rows]) - int(ptr[TM]) > E_CAP
    A = {(0, 0): a00, (0, 1): rand_csr(rng, rows, blk, 0.02), (0, 2): csr_from_rows(rows, blk, [[]] * rows, rng),
         (0, 3): rand_csr(rng, rows, 300, 0.05)}
    k, m = 3 * blk + 300, 200
    B = blocks_of(rng.uniform(-1, 1, (k, m)), blk, LAYOUTS["mixed"])
    return A, B, rows, k, m, blk


def test_segment_capacity_and_the_global_window(sess):
    rng = np.random.default_rng(664)
    A, B, n, k, m, blk = capacity_operands(rng)
    got = run_route(sess, A, B, n, k, m, blk, "pipelined")
    check(got, A, B, n, k, m, blk, rng, samples=400)
    G, S = O.assemble(got, n, m, blk), sparse_sum_bound(A, B, n, k, m, blk)
    for r in (0, 5, 16, 17, 18, 32, 37, 255, 256, 499):                                  # every row the segments were built from
        for j, x in enumerate(exact_sparse_entries(A, B, n, k, m, blk, [(r, j) for j in range(m)])):
            assert within(G[r, j], x, S[r, j]), (r, j)
    again = run_route(sess, A, B, n, k, m, blk, "pipelined")
    same_bits(got, again)                                                                 # deterministic
    fused = run_route(sess, A, B, n, k, m, blk, "fused", spmm_algo=1)
    same_bits(got, fused)             # sorted rows, no dense partial: the same FMA chain per element in both kernels
    same_bits(fused, run_route(sess, A, B, n, k, m, blk, "fused", spmm_algo=1))


# ------------------------------------------------------------------------------------------------ layouts
def test_densified_sparse_right_blocks(sess):
    """Sparse x sparse with the right density > 0.1 multiplies the left's stored entries with B.toDense (LocalMatrix.scala:906-907)."""
    rng = np.random.default_rng(11)
    n, k, m, blk = 512, 4 * 256, 160, 256
    A = sparse_rows(rng, n, k, 256, 0.03)
    Bf = rng.uniform(-1, 1, (k, m)) * (rng.random((k, m)) < 0.3)
    B = {key: dense(b.to_numpy(), False).toSparse() for key, b in blocks_of(Bf, blk).items()}
    got = run_route(sess, A, B, n, k, m, blk, "pipelined")
    check(got, A, B, n, k, m, blk, rng)


def test_unaligned_right_blocks_take_the_fused_kernel(sess):
    from tests.test_gpu_unaligned import adopt_unaligned
    rng = np.random.default_rng(12)
    n, k, m, blk = 512, 4 * 256, 200, 256
    A = sparse_rows(rng, n, k, blk, 0.03)
    B = blocks_of(rng.uniform(-1, 1, (k, m)), blk, LAYOUTS["mixed"])
    dB, keep = adopt_unaligned(sess, B)
    assert all(dB.block_device_ptr(*key) % 16 == 8 for key in B)
    got = run_route(sess, A, B, n, k, m, blk, "fused", aligned=False, dB=dB)
    check(got, A, B, n, k, m, blk, rng)
    del dB, keep


def test_unsorted_rows(sess):
    rng = np.random.default_rng(13)
    n, k, m, blk = 512, 4 * 256, 130, 256
    A = sparse_rows(rng, n, k, blk, 0.06, sort=False)
    assert any(np.any(np.diff(a.rowIndices[a.colPtrs[r]:a.colPtrs[r + 1]]) < 0) for a in A.values() for r in range(a.numRows))
    B = blocks_of(rng.uniform(-1, 1, (k, m)), blk, LAYOUTS["row"])
    for route, algo in (("pipelined", 0), ("fused", 1)):
        check(run_route(sess, A, B, n, k, m, blk, route, spmm_algo=algo), A, B, n, k, m, blk, rng)


@pytest.mark.parametrize("route", ["pipelined", "fused", "csc", "csc+csr"])
def test_csc_left_blocks_and_duplicate_indices(sess, route):
    """CSC blocks (per-pair scatter with fp64 atomics: held to the bound only), alone and next to CSR blocks in one output block;
    rows that repeat a column index (the reference adds both terms)."""
    rng = np.random.default_rng(14 + len(route))
    n, k, m, blk = 512, 4 * 256, 96, 256
    A = sparse_rows(rng, n, k, blk, 0.04, dups=0.3)
    if route.startswith("csc"):
        A = {key: to_csc(a) if route == "csc" or key[1] % 2 == 0 else a for key, a in A.items()}
    B = blocks_of(rng.uniform(-1, 1, (k, m)), blk, LAYOUTS["mixed"])
    got = run_route(sess, A, B, n, k, m, blk, "csc" if route.startswith("csc") else route, spmm_algo=1 if route == "fused" else 0)
    if route == "csc+csr":
        assert plan_routes(A, B)[1] == {"csc", "pipelined"}
    check(got, A, B, n, k, m, blk, rng)


def test_duplicate_indices_on_the_per_pair_csr_kernel(sess):
    rng = np.random.default_rng(15)
    n, k, m, blk = 1100, 2048 + 100, 40, 2048
    A = sparse_rows(rng, n, k, blk, 0.02, dups=0.5)
    B = blocks_of(rng.uniform(-1, 1, (k, m)), blk)
    got = run_route(sess, A, B, n, k, m, blk, "csr")
    check(got, A, B, n, k, m, blk, rng)


# ------------------------------------------------------------------------------------------------ partial sums
@pytest.mark.parametrize("spmm_algo", [0, 1])
def test_dense_csc_and_csr_partials_in_one_output_block(sess, spmm_algo):
    """DMMA writes the dense partial, the per-pair CSC kernel adds its pairs, the fused / pipelined kernel accumulates on top."""
    rng = np.random.default_rng(16 + spmm_algo)
    n, k, m, blk = 500, 5 * 256, 130, 256
    A = sparse_rows(rng, n, k, blk, 0.04)
    for i in range(2):
        A[(i, 0)] = dense(rng.uniform(-1, 1, (A[(i, 0)].numRows, 256)), i == 1)
        A[(i, 1)], A[(i, 4)] = to_csc(A[(i, 1)]), to_csc(A[(i, 4)])
    B = blocks_of(rng.uniform(-1, 1, (k, m)), blk, LAYOUTS["mixed"])
    launches, routes = plan_routes(A, B, spmm_algo)
    assert routes == ({"csc", "pipelined"} if spmm_algo == 0 else {"csc", "fused"})
    got, st = multiply(sess, A, B, n, k, m, blk, spmm_algo=spmm_algo)
    assert st["kernel_launches"] == launches and st["tc_gemm_launches"] == 0
    check(got, A, B, n, k, m, blk, rng)


@pytest.fixture(scope="module")
def big_mixed():
    """4096^3 at blk 1024: block rows 0-1 dense, 2-3 all CSR.  The dense rows alone are 2^36 flops, far above the 2^33 at which
    the auto selection takes the Ozaki-II engine."""
    rng = np.random.default_rng(17)
    n = k = m = 4096
    blk = 1024
    Ad = rng.uniform(-1, 1, (2 * blk, k))
    A = {(i, kb): dense(Ad[i * blk:(i + 1) * blk, kb * blk:(kb + 1) * blk], kb % 2 == 1) for i in range(2) for kb in range(4)}
    A.update({(i, kb): rand_csr(rng, blk, blk, 0.01) for i in (2, 3) for kb in range(4)})
    Bf = rng.uniform(-1, 1, (k, m))
    return A, Ad, Bf, blocks_of(Bf, blk, LAYOUTS["mixed"]), n, k, m, blk, rng


def test_ozaki2_dense_rows_next_to_sparse_rows(sess, big_mixed):
    A, Ad, Bf, B, n, k, m, blk, rng = big_mixed
    got, st = multiply(sess, A, B, n, k, m, blk, gemm_algo=0)
    assert st["tc_gemm_launches"] == 1 and st["tc_moduli"] == moduli_for(k)
    G = check(got, A, B, n, k, m, blk, rng, samples=100, rows=slice(2 * blk, n))        # sparse rows: the sparse bound
    D = G[:2 * blk]
    alpha = alpha_of(moduli_for(k), k)
    ref = Ad @ Bf
    op = oz2_bound(Ad, Bf, alpha, ref)
    assert np.all(np.abs(D - ref) <= op + fp64_dot_bound(Ad, Bf))
    pos = [(int(rng.integers(2 * blk)), int(rng.integers(m))) for _ in range(24)] + [(0, 0), (2 * blk - 1, m - 1), (1023, 1024)]
    for (i, j), x in zip(pos, exact_entries(Ad, Bf, pos)):
        assert within(D[i, j], x, op[i, j]), (i, j)


def test_inf_in_a_dense_block_leaves_the_sparse_rows_bit_for_bit(sess, big_mixed):
    A, Ad, Bf, B, n, k, m, blk, rng = big_mixed
    before, _ = multiply(sess, A, B, n, k, m, blk, gemm_algo=0)
    Ad2 = Ad.copy()
    Ad2[5, 7] = np.inf
    A2 = dict(A)
    A2[(0, 0)] = dense(Ad2[:blk, :blk], False)
    got, st = multiply(sess, A2, B, n, k, m, blk, gemm_algo=0)
    assert st["tc_gemm_launches"] == 1
    for key, v in got.items():
        if key[0] >= 2:
            assert np.array_equal(v.values, before[key].values), key
    D = O.assemble(got, n, m, blk)[:2 * blk]
    with np.errstate(invalid="ignore", over="ignore"):
        ref = Ad2 @ Bf
        fin = np.isfinite(ref)
        assert np.array_equal(D[~fin], ref[~fin], equal_nan=True) and (~fin).sum() == m
        assert np.all(np.abs(D - ref)[fin] <= 2 * fp64_dot_bound(np.where(np.isfinite(Ad2), Ad2, 0), Bf)[fin])


# ------------------------------------------------------------------------------------------------ values
def value_operands(rng, n, blk):
    """Rows 0-29 hold the special cases, the other rows random entries outside the special k range [900, 990):
      0-9   wide range 1e+-150 inside one row             10-19 products and sums in the sub-normal range
      20-21 products that overflow to +inf / -inf         22    +inf and -inf terms (-> NaN)
      23-26 exact cancellation to 0
      27    a stored 0.0 facing +inf (-> NaN)             28    a stored 2.0 facing +inf (-> +inf)
    B rows 970-989 hold NaN and +-inf and no stored entry faces them; B is dyadic with 20-bit mantissas so that the
    cancelling products are exact."""
    k, m = 1024, 130
    Bf = np.round(rng.uniform(-1, 1, (k, m)) * 2 ** 20) / 2 ** 20
    Bf[900:910] = np.abs(Bf[900:910]) * 1e200 + 1e200                     # overflow partners, all positive
    Bf[950] = Bf[951]
    Bf[961], Bf[962] = -np.inf, np.inf
    Bf[960, 5] = np.inf
    Bf[970:980, ::3], Bf[980:990, 1::3], Bf[975:985, 2::3] = np.nan, np.inf, -np.inf
    row_cols, vals = [], []
    for r in range(n):
        if r < 10:
            c = rng.choice(900, 40, replace=False)
            v = rng.choice([-1, 1], 40) * 10.0 ** rng.uniform(-150, 150, 40)
        elif r < 20:
            c = rng.choice(900, 30, replace=False)
            v = rng.uniform(-1, 1, 30) * 1e-310
        elif r < 22:
            c = np.arange(900, 910)
            v = np.full(10, 1e200) * [1, -1][r - 20]
        elif r == 22:
            c, v = np.array([961, 962, 3]), np.array([1.0, 1.0, 0.5])         # +inf and -inf terms
        elif r < 27:
            c, v = np.array([950, 951]), np.array([3.0, -3.0]) * (r - 22)
        elif r < 29:
            c, v = np.array([960, 10]), np.array([0.0 if r == 27 else 2.0, 0.5])
        else:
            c = np.flatnonzero(rng.random(900) < 0.03)
            v = rng.uniform(-1, 1, c.size)
        o = np.argsort(c, kind="stable")                                      # sorted rows: pipelined == fused bit for bit
        row_cols.append(c[o])
        vals.append(v[o])
    Ad = csr_from_rows(n, k, row_cols, rng, vals)
    return Ad, Bf, k, m


def split(a, blk):
    """A whole CSR matrix cut into CSR blocks of blk x blk (entry order kept)."""
    out = {}
    rows = np.repeat(np.arange(a.numRows), np.diff(a.colPtrs))
    for bi in range(-(-a.numRows // blk)):
        for kb in range(-(-a.numCols // blk)):
            r0, c0 = bi * blk, kb * blk
            nr, nc = min(blk, a.numRows - r0), min(blk, a.numCols - c0)
            sel = (rows >= r0) & (rows < r0 + nr) & (a.rowIndices >= c0) & (a.rowIndices < c0 + nc)
            out[(bi, kb)] = csr_from_rows(nr, nc, [a.rowIndices[sel & (rows == r0 + r)] - c0 for r in range(nr)], None,
                                          [a.values[sel & (rows == r0 + r)] for r in range(nr)])
    return out


@pytest.mark.parametrize("route", ["pipelined", "fused", "csr", "csc"])
def test_extreme_values_and_unreferenced_non_finite_rows(sess, route):
    rng = np.random.default_rng(18)
    n, blk = (1100, 2048) if route == "csr" else (512, 256)
    Ad, Bf, k, m = value_operands(rng, n, blk)
    A = split(Ad, blk)
    if route == "csc":
        A = {key: to_csc(a) for key, a in A.items()}
    B = blocks_of(Bf, blk, LAYOUTS["mixed"])
    algo = 1 if route == "fused" else 0
    got = run_route(sess, A, B, n, k, m, blk, route, spmm_algo=algo)
    G = check(got, A, B, n, k, m, blk, rng, samples=100)
    with np.errstate(invalid="ignore"):
        assert np.all(np.isfinite(G[29:])) and np.all(np.isfinite(G[:20]))   # the NaN / inf rows of B never reach C
        assert np.all(G[20] == np.inf) and np.all(G[21] == -np.inf) and np.all(np.isnan(G[22]))
        assert np.all(G[23:27] == 0.0) and np.isnan(G[27, 5]) and G[28, 5] == np.inf
        assert np.isfinite(np.delete(G[27:29], 5, axis=1)).all()
        assert np.any((np.abs(G[10:20]) < 2.0 ** -1022) & (G[10:20] != 0))             # sub-normal results
    if route != "csc":                                                                 # deterministic routes
        same_bits(got, run_route(sess, A, B, n, k, m, blk, route, spmm_algo=algo))
    if route == "pipelined":
        same_bits(got, run_route(sess, A, B, n, k, m, blk, "fused", spmm_algo=1))


def test_spmv_ignores_unreferenced_non_finite_rows(sess):
    """n = 1 (LocalMatrix.multiplySparseMatDenseVec) reads B only where a stored entry faces it, like gemmsdd."""
    rng = np.random.default_rng(19)
    n, blk = 512, 256
    Ad, Bf, k, _ = value_operands(rng, n, blk)
    A = split(Ad, blk)
    B = blocks_of(Bf[:, 3:4], blk)                       # column 3: NaN at rows 970-979 and 975-984, no entry faces them
    assert np.isnan(Bf[970:980, 3]).all()
    got = run_route(sess, A, B, n, k, 1, blk, "fused")
    G = check(got, A, B, n, k, 1, blk, rng)
    assert np.isfinite(np.delete(G[:, 0], [20, 21, 22])).all()


# ------------------------------------------------------------------------------------------------ mr_grid_multiply_rows
@pytest.mark.parametrize("pr,pc", [(1, 1), (2, 1), (2, 2)])
@pytest.mark.parametrize("kind", ["sparse", "dense"])
def test_grid_multiply_rows_on_one_device(kind, pr, pc):
    """Every virtual rank (r, c) of a pr x pc grid on device 0: its share of C = A B through mr_grid_multiply_rows, with B's
    column slabs taken straight from the tensors.  The union must be the resident multiply, bit for bit."""
    import torch
    from matrel_b200.dataset import grid_multiply_rows
    from matrel_b200.distributed import GridPlan, ShardedMatrix
    rng = np.random.default_rng(pr * 10 + pc)
    n, k, m, blk = 700, 900, 600, 256                                    # ragged in all three dimensions
    world = pr * pc
    planB, planC = GridPlan(world, k, m, blk, pr, pc), GridPlan(world, n, m, blk, pr, pc)
    if kind == "sparse":
        A = sparse_rows(rng, n, k, blk, 0.03)
    else:
        A = blocks_of(rng.uniform(-1, 1, (n, k)), blk, LAYOUTS["mixed"])
    with mb.MatfastSession(device=0, gemm_algo=1) as s:
        s.set_option("gemm_variant", 1)
        Bs = [ShardedMatrix.rand(s, planB, rank, 43, torch.device("cuda", 0)) for rank in range(world)]
        s.sync()
        Bfull = {}
        for b in Bs:
            Bfull.update({key: O.DenseMatrix(v.numRows, v.numCols, v.values, v.isTransposed) for key, v in from_dataset(b.dataset).items()})
        assert sorted(Bfull) == [(i, j) for i in range(planB.nbr) for j in range(planB.nbc)]
        dA = to_dataset(s, A)
        resident = from_dataset(dA.matrixMultiply(n, k, to_dataset(s, Bfull), k, m, blk))
        union = {}
        for rank in range(world):
            r, c = planC.coords(rank)
            col = [Bs[planB.rank_of(rr, c)].slab.data_ptr() for rr in range(pr)]
            s.reset_stats()
            out = grid_multiply_rows(s, dA.filter_blocks(pr, r), n, k, Bs[rank].sharded, col)
            assert (s.stats()["p2p_bytes"] > 0) == (pr > 1)
            ids = sorted(out.block_ids())
            assert ids == sorted(planC.owned(rank)), rank
            base = out.block_device_ptr(*ids[0]) - planC.slot(*ids[0]) * planC.slot_elems * 8
            assert all(out.block_device_ptr(i, j) == base + planC.slot(i, j) * planC.slot_elems * 8 for i, j in ids)
            union.update(from_dataset(out))
        assert sorted(union) == sorted(resident)
        for key, v in resident.items():
            assert np.array_equal(union[key].to_numpy(), v.to_numpy()), key
        if pr > 1:                                                       # the three argument checks
            with pytest.raises(mb.IllegalArgumentException) as e:
                grid_multiply_rows(s, dA, n, k, Bs[0].sharded, [b.slab.data_ptr() for b in Bs[:pr]])
            assert "is not in a block row of rank (0, 0)" in N.last_error() and N.last_error() in str(e.value)
            with pytest.raises(mb.IllegalArgumentException) as e:
                grid_multiply_rows(s, dA.filter_blocks(pr, 0), n, k + 1, Bs[0].sharded, [b.slab.data_ptr() for b in Bs[:pr]])
            assert N.last_error() == f"requirement failed: Matrix dimension not match, leftColNum = {k + 1}, rightRowNum = {k}"
            from matrel_b200.dataset import adopt_sharded
            bt = adopt_sharded(s, k, m, blk, pr, pc, 0, 0, Bs[0].slab.data_ptr(), True)
            with pytest.raises(Exception):
                grid_multiply_rows(s, dA.filter_blocks(pr, 0), n, k, bt, [b.slab.data_ptr() for b in Bs[:pr]])
            assert "flag-transposed" in N.last_error()
        del Bs

"""Edge tests of the dense element-wise, scalar, slicing and aggregate kernels (ew.cu) against exact references
(tests/dense_ew_ref.py), element by element, at the shapes that reach each launch path:

  ew_flat_kernel / map_kernel   the 4-way unrolled grid-stride loop, its remainder loop and the scalar tail of odd element counts;
                                the grid cap of 65535 CTAs (a 12000 x 12000 block)
  ew_tiled_kernel               layout-mixing add / multiply / divide, the materialising transpose, the rank-one update
  axis_sum_kernel               "kept fast" (rowSum of a column-major block, colSum of a row-major one) with slow extents above
                                AGG_SLOW = 256, where CTAs add atomically into one entry; "kept slow" with fast extents of 128 and
                                more (the 4-way sweep) and above AGG_SWEEP = 1024 (a second sweep)
  scalar_sum_kernel             sum and trace, the grid cap of 1024 CTAs (blocks above 2048^2 elements)
  extract_lines_kernel          project and selection of both layouts
  every launcher but trace's     more than 65535 blocks in one call (split over gridDim.y); trace reads only the diagonal blocks

Element-wise operations, scalar maps, power(2), power(0.5), copies and slices are single IEEE operations per element and are
compared bit for bit with the oracle.  Aggregates of integer-valued data are exact in every summation order and are compared bit
for bit; aggregates of full-mantissa data with heavy cancellation are held to gamma_(n-1) sum |x| of each entry, the bound of any
order (the dense sums use fp64 atomics).  There is no check relative to a block's largest entry."""
import ctypes
import math

import numpy as np
import pytest

import matrel_b200 as mb
from oracle import matrel_oracle as O
from tests import dense_ew_ref as R
from tests.util import assert_same_dataset, from_dataset, to_dataset

pytestmark = pytest.mark.gpu

AGG = {"row": "rowSum", "col": "colSum", "sum": "sum", "trace": "trace"}


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


def block(a, rowmajor):
    a = np.asarray(a, dtype=np.float64)
    return O.DenseMatrix(a.shape[0], a.shape[1], np.ascontiguousarray(a if rowmajor else a.T).reshape(-1), bool(rowmajor))


def grid(hs, ws, fill, rowmajor):
    """Blocks (i, j) of hs[i] x ws[j] values fill(h, w), row-major where rowmajor(i, j)."""
    return {(i, j): block(fill(h, w), rowmajor(i, j)) for i, h in enumerate(hs) for j, w in enumerate(ws)}


def integers(rng):
    return lambda h, w: rng.integers(-2 ** 20, 2 ** 20, (h, w)).astype(np.float64)


def full_mantissas(rng):
    return lambda h, w: R.cancelling(rng, h, w) if w > 1 else rng.uniform(-1, 1, (h, w)) * 2.0 ** rng.integers(0, 40, (h, w))


def specials(rng, h, w):
    """Full mantissas in [-1e3, 1e3] with subnormals, +-0.0, NaN, +-Inf and 1.5e308 (near overflow) sprinkled in.  A line
    whose sum class would depend on the summation order (an Inf next to finite terms that may overflow the other way) loses its
    -Inf, so every order gives the class sum_class names."""
    a = rng.uniform(-1e3, 1e3, (h, w))
    u = rng.random((h, w))
    for lo, hi, v in ((0.0, 0.05, None), (0.05, 0.08, 0.0), (0.08, 0.11, -0.0), (0.11, 0.1105, np.nan),
                      (0.1105, 0.111, np.inf), (0.111, 0.1115, -np.inf), (0.1115, 0.1125, 1.5e308)):
        sel = (u >= lo) & (u < hi)
        a[sel] = rng.uniform(-1, 1, int(sel.sum())) * 2.0 ** -1060 if v is None else v
    for _ in range(4):
        fixed = 0
        for lines in (a, a.T):  # rows, then columns (views: the fix lands in a)
            for line in lines:
                try:
                    R.sum_class(line)
                except ValueError:
                    line[np.isneginf(line)] = 1.0
                    fixed += 1
        if not fixed:
            return a
    raise AssertionError("special values: order-dependent lines left")


def split(a, hs, ws, rowmajor):
    """The blocks hs[i] x ws[j] of the matrix a."""
    r = np.cumsum([0] + hs)
    c = np.cumsum([0] + ws)
    return {(i, j): block(a[r[i]:r[i + 1], c[j]:c[j + 1]], rowmajor(i, j)) for i in range(len(hs)) for j in range(len(ws))}


LAYOUTS = {
    "col": (lambda i, j: False, lambda i, j: False),              # every block column-major: the flat path
    "row": (lambda i, j: True, lambda i, j: True),                # every block row-major: the tiled path, both operands staged
    "mixed": (lambda i, j: (i + j) % 2 == 1, lambda i, j: (i + j) % 2 == 0),
}


def exact(got, want):
    """Same block ids, types, shapes and flags, and the same bits: signed zeros included, NaN payloads aside."""
    assert_same_dataset(got, want, exact_storage=True)
    for key, w in want.items():
        assert np.array_equal(R.bits(got[key].values), R.bits(w.values)), key


def check_elementwise(s, A, B, n, m, blk):
    """add / multiply / divide (B may lack blocks of A: the outer join passes them through, the inner joins drop them), scalar
    add / multiply, power(2), power(0.5), the materialising transpose, all bit for bit."""
    dA, dB = to_dataset(s, A), to_dataset(s, B)
    exact(from_dataset(dA.addElement(n, m, dB, n, m, blk)), O.add_element(A, n, m, B, n, m, blk))
    exact(from_dataset(dA.multiplyElement(n, m, dB, n, m, blk)), O.multiply_element(A, n, m, B, n, m, blk))
    exact(from_dataset(dA.divideElement(n, m, dB, n, m, blk)), O.divide_element(A, n, m, B, n, m, blk))
    exact(from_dataset(dA.addScalar(0.1)), O.add_scalar(A, 0.1))
    exact(from_dataset(dA.multiplyScalar(-1.0 / 3.0)), O.multiply_scalar(A, -1.0 / 3.0))
    exact(from_dataset(dA.power(2.0)), O.power(A, 2.0))
    exact(from_dataset(dA.power(0.5)), O.power(A, 0.5))
    want = {k: O.DenseMatrix(v.numRows, v.numCols, v.toArray()) for k, v in O.transpose(A).items()}
    exact(from_dataset(dA.t().materialize()), want)


def check_slices(s, A, n, m, blk, rows, cols):
    d = to_dataset(s, A)
    for i in rows:
        exact(from_dataset(d.project(n, m, blk, True, i)), O.project(A, n, m, blk, True, i))
    for j in cols:
        exact(from_dataset(d.project(n, m, blk, False, j)), O.project(A, n, m, blk, False, j))
    for i in rows:
        for j in cols:
            exact(from_dataset(d.selection(n, m, blk, i, j)), O.selection(A, n, m, blk, i, j))


def check_aggregates(s, A, n, m, integer, ops=("row", "col", "sum", "trace")):
    """Every output entry: integer data bit for bit against the exact sum, other data within the bound of any order."""
    d = to_dataset(s, A)
    for op in ops:
        if op == "trace" and (n != m or any(i == j and b.numRows != b.numCols for (i, j), b in A.items())):
            continue  # trace needs a square matrix of square diagonal blocks
        got = from_dataset(getattr(d, AGG[op])(n, m))
        want = R.lines(op, A)
        assert sorted(got) == sorted(want), op
        for key, T in want.items():
            g = got[key].values
            assert g.size == T.shape[0]
            if integer:
                assert np.array_equal(R.bits(g), R.bits(R.int_sums(T))), (op, key)
            else:
                ok = R.sums_within_bound(g, T)
                assert ok.all(), (op, key, np.flatnonzero(~ok)[:10])


SHAPES = {
    "1x1": ([1], [1]),
    "1xN": ([1], [4096]),
    "Nx1": ([4096], [1]),
    "small": ([31, 127], [128, 257]),
    "tall-wide": ([1025, 1], [1, 1025]),      # 1025 x 1 and 1 x 1025 blocks next to 1 x 1 and 1025 x 1025 ones
    "sweeps": ([257, 128], [1025, 31]),
    "square": ([4096], [4096]),               # sum above 2048^2 elements: the 1024-CTA cap
    "diag": ([1, 31, 127, 128], [1, 31, 127, 128]),
}


def offsets(ext):
    """A few global indices: each block's first and last line, and an interior one."""
    out, at = set(), 0
    for e in ext:
        out |= {at, at + e - 1, at + e // 2}
        at += e
    return sorted(out)


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("shape", list(SHAPES))
def test_shapes(sess, shape, layout):
    """Each shape of SHAPES under each layout mix: the element-wise operations, slices (bit for bit) and the four aggregates
    (integer data bit for bit, cancelling full-mantissa data within the summation bound).  'col' runs ew_flat_kernel, 'row' and
    'mixed' ew_tiled_kernel; the aggregates reach both axis_sum_kernel shapes with slow extents 257 .. 4096 (kept fast: several
    CTAs per entry) and fast extents 128 .. 4096 (kept slow: the 4-way sweep, and a second sweep above 1024)."""
    hs, ws = SHAPES[shape]
    la, lb = LAYOUTS[layout]
    rng = np.random.default_rng([len(hs), sum(hs), sum(ws), len(layout)])
    n, m, blk = sum(hs), sum(ws), max(hs + ws)
    A = grid(hs, ws, full_mantissas(rng), la)
    B = grid(hs, ws, lambda h, w: rng.uniform(-4, 4, (h, w)) * 2.0 ** rng.integers(-30, 30, (h, w)), lb)
    if len(B) > 1:
        del B[max(B)]  # an absent block
    check_elementwise(sess, A, B, n, m, blk)
    # slices of block (0, 0) (project / selection find blocks by blkSize, which these grids do not share)
    check_slices(sess, {(0, 0): A[(0, 0)]}, hs[0], ws[0], blk, offsets(hs[:1]), offsets(ws[:1]))
    check_aggregates(sess, grid(hs, ws, integers(rng), la), n, m, integer=True)
    check_aggregates(sess, A, n, m, integer=False)


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_tall_and_wide_blocks_without_a_corner(sess, layout):
    """A batch of a 1025 x 1 block (0, 0) and a 1 x 1025 block (1, 1) and nothing else: max_rows and max_cols come from
    different blocks, and no block is as large as both, so the flat, tiled and axis-sum grids are sized from the two maxima
    and must decode each block's tiles from them.  Element-wise operations, maps and the materialising transpose bit for bit;
    rowSum, colSum and sum of integer data bit for bit, of cancelling full-mantissa data within the summation bound."""
    la, lb = LAYOUTS[layout]
    rng = np.random.default_rng([19, len(layout)])
    shapes = {(0, 0): (1025, 1), (1, 1): (1, 1025)}
    A = {k: block(full_mantissas(rng)(h, w), la(*k)) for k, (h, w) in shapes.items()}
    B = {k: block(rng.uniform(-4, 4, (h, w)) * 2.0 ** rng.integers(-30, 30, (h, w)), lb(*k)) for k, (h, w) in shapes.items()}
    n = m = 1026
    check_elementwise(sess, A, B, n, m, 1025)
    I = {k: block(integers(rng)(h, w), la(*k)) for k, (h, w) in shapes.items()}
    check_aggregates(sess, I, n, m, integer=True, ops=("row", "col", "sum"))
    check_aggregates(sess, A, n, m, integer=False, ops=("row", "col", "sum"))


def test_slices_of_a_block_grid(sess):
    """project / selection over a uniform grid of 257-blocks with ragged edges (600 = 257 + 257 + 86), mixed layouts."""
    rng = np.random.default_rng(11)
    hs, ws, blk = [257, 257, 86], [257, 31], 257
    A = grid(hs, ws, full_mantissas(rng), LAYOUTS["mixed"][0])
    check_slices(sess, A, sum(hs), sum(ws), blk, offsets(hs), offsets(ws))


def test_special_values(sess):
    """+-0.0, subnormals, NaN, +-Inf, 1.5e308 and 0/0 in both layouts: element-wise operations, maps and copies bit for bit; the
    aggregates in the non-finite class every summation order gives, finite entries within the bound."""
    rng = np.random.default_rng(12)
    hs, ws = [31, 257], [128, 1025]
    n, m, blk = sum(hs), sum(ws), 1025
    a = specials(rng, n, m)
    b = specials(rng, n, m)
    b[(a == 0.0) & (rng.random(a.shape) < 0.5)] = -0.0  # 0/0
    A = split(a, hs, ws, LAYOUTS["mixed"][0])
    B = split(b, hs, ws, LAYOUTS["mixed"][1])
    for lines in (a, a.T):
        classes = {R.sum_class(line) for line in lines}
        assert classes == {"nan", "+inf", "-inf", "finite"}, classes
    check_elementwise(sess, A, B, n, m, blk)
    check_aggregates(sess, A, n, m, integer=False, ops=("row", "col", "sum"))
    check_slices(sess, {(0, 0): A[(0, 1)]}, 31, 1025, 1025, [0, 17, 30], [0, 500, 1024])  # a 31 x 1025 row-major block


def pow_inputs(rng):
    xs = sorted({x for x, _, _ in R.SPECIAL} | {0.5, -0.5, 3.0, -3.0, 2.0 ** -1074, 1e308, -1e-300}, key=repr)
    rand = np.concatenate([rng.uniform(0, 4, 900), -rng.uniform(0, 4, 100), 2.0 ** rng.uniform(-1070, 1020, 200)])
    return np.concatenate([np.array(xs), rand])


@pytest.mark.parametrize("p", [-1.3, 3.0, -2.0, 0.25, 1.0 / 3.0, 7.5, -0.5, 1.5, 2.0, 0.5, 1.0, 0.0, -0.0,
                               math.inf, -math.inf, math.nan])
def test_power(sess, p):
    """power(p) against java.lang.Math.pow: where x or p is special (0, +-Inf, NaN, +-1, p in {0, 1}) or the result is NaN, bit
    for bit (NaN as NaN); otherwise within 2 ulp, overflow and underflow included (CUDA documents 2 ulp for double pow), and
    bit for bit for p = 2 and 0.5, which take the exact closed forms.  The values are split over a column-major block and a
    row-major one of odd length, which reaches the scalar tail of map_kernel."""
    rng = np.random.default_rng(13)
    x = pow_inputs(rng)
    A = {(0, 0): block(x[:613].reshape(613, 1), False), (0, 1): block(x[613:].reshape(1, -1), True)}
    assert A[(0, 1)].values.size % 2 == 1
    got = from_dataset(to_dataset(sess, A).power(p))
    for k, a in A.items():
        g = got[k].values
        assert (got[k].numRows, got[k].numCols, got[k].isTransposed) == (a.numRows, a.numCols, a.isTransposed)
        want = np.array([R.java_pow(v, p) for v in a.values])
        special = np.array([v == 0.0 or not math.isfinite(v) or abs(v) == 1.0 or not math.isfinite(p) or p in (0.0, 1.0) or
                            math.isnan(w) for v, w in zip(a.values, want)])
        if p in (2.0, 0.5):
            special[:] = True
        bad = [i for i in np.flatnonzero(special) if R.bits(g[i])[0] != R.bits(want[i])[0]]
        assert not bad, [(a.values[i], g[i], want[i]) for i in bad[:8]]
        far = [i for i, d in zip(np.flatnonzero(~special), R.ulp_distance(g[~special], want[~special])) if d > 2]
        assert not far, [(a.values[i], g[i], want[i]) for i in far[:8]]


def vector(rng, hs):
    return {(i, 0): block(rng.standard_normal((h, 1)) * 2.0 ** rng.integers(-20, 20, (h, 1)), False) for i, h in enumerate(hs)}


@pytest.mark.parametrize("layout", ["col", "row", "mixed"])
def test_rank_one_update(sess_intended, layout):
    """A + v v^T (intended semantics) over square blocks 1 .. 257 with ragged edges: a + (x y), both operations rounded, bit for
    bit.  Element (0, 0) is x = y = 1 + 2^-30 and a = -(1 + 2^-29): two roundings give 0.0, a fused multiply-add 2^-60."""
    rng = np.random.default_rng(14 + len(layout))
    hs = [1, 31, 257, 128] if layout != "mixed" else [127, 257]
    n, blk = sum(hs), max(hs)
    A = grid(hs, hs, lambda h, w: rng.standard_normal((h, w)) * 2.0 ** rng.integers(-20, 20, (h, w)), LAYOUTS[layout][0])
    v = vector(rng, hs)
    a00 = R.dense_array(A[(0, 0)]).copy()
    a00[0, 0] = -(1.0 + 2.0 ** -29)
    A[(0, 0)] = block(a00, A[(0, 0)].isTransposed)
    x0 = v[(0, 0)].values.copy()
    x0[0] = 1.0 + 2.0 ** -30
    v[(0, 0)] = O.DenseMatrix(hs[0], 1, x0)
    s = sess_intended
    got = from_dataset(to_dataset(s, A).matrixRankOneUpdate(n, n, to_dataset(s, v), n, 1, blk))
    want = O.rank_one_update(A, n, n, v, n, 1, blk, compat_bugs=False)
    assert want[(0, 0)].values[0] == 0.0
    exact(got, want)


def test_rank_one_update_compat(sess):
    """The reference's rankOneAdd (compat_bugs): x_r y_c written at A's storage index, over blocks of both layouts.  The
    reference's requires admit only 1-row datasets, so the call names 1 x n dimensions over larger blocks."""
    rng = np.random.default_rng(15)
    hs = [31, 257, 128]
    A = grid(hs, hs, lambda h, w: rng.standard_normal((h, w)), LAYOUTS["mixed"][0])
    v = vector(rng, hs)
    got = from_dataset(to_dataset(sess, A).matrixRankOneUpdate(1, sum(hs), to_dataset(sess, v), 1, 1, max(hs)))
    exact(got, O.rank_one_update(A, 1, sum(hs), v, 1, 1, max(hs), compat_bugs=True))


def test_block_above_the_flat_grid_cap(sess):
    """One 12000 x 12000 block (1.15 GB): 72 M double2 vectors exceed the 65535 x 256 x 4 a capped flat grid covers in one
    unrolled pass, so the remainder loop runs; sum runs on the 1024-CTA cap.  Element-wise operations and maps bit for bit,
    aggregates of integer data bit for bit; the materialising transpose on the tiled path (140625 tiles)."""
    rng = np.random.default_rng(16)
    n = 12000
    a = rng.integers(-1000, 1000, (n, n)).astype(np.float64)
    A = {(0, 0): block(a, False)}
    del a
    B = {(0, 0): O.DenseMatrix(n, n, rng.uniform(0.5, 2.0, n * n))}
    dA, dB = to_dataset(sess, A), to_dataset(sess, B)
    for fn, want in ((lambda: dA.addElement(n, n, dB, n, n, n), lambda: O.add_element(A, n, n, B, n, n, n)),
                     (lambda: dA.divideElement(n, n, dB, n, n, n), lambda: O.divide_element(A, n, n, B, n, n, n)),
                     (lambda: dB.multiplyScalar(-3.0), lambda: O.multiply_scalar(B, -3.0)),
                     (lambda: dB.power(0.5), lambda: O.power(B, 0.5))):
        exact(from_dataset(fn()), want())
    got = from_dataset(dA.t().materialize())[(0, 0)]
    assert not got.isTransposed and np.array_equal(R.dense_array(got), R.dense_array(A[(0, 0)]).T)
    del dB, B, got
    check_aggregates(sess, A, n, n, integer=True)


def test_more_than_65535_blocks(sess, sess_intended):
    """A 260 x 260 matrix at blkSize 1 (67,600 blocks, built with fromDense from C- and F-ordered arrays): the element-wise,
    map, copy, rank-one and rowSum / colSum / sum launches are split over gridDim.y (trace and project read only 260 blocks
    here; test_project_of_more_than_65535_blocks splits project).  Element-wise operations, maps, copies and the rank-one
    update bit for bit; integer aggregates bit for bit."""
    rng = np.random.default_rng(17)
    n = 260
    a = rng.integers(-2 ** 20, 2 ** 20, (n, n)).astype(np.float64)
    b = rng.uniform(-1, 1, (n, n)) * 2.0 ** rng.integers(-30, 30, (n, n))
    dA = sess.fromDense(np.asfortranarray(a), 1)   # column-major 1 x 1 blocks
    dB = sess.fromDense(np.ascontiguousarray(b), 1)  # row-major 1 x 1 blocks
    dBf = sess.fromDense(np.asfortranarray(b), 1)
    assert len(dA.block_ids()) == n * n and dB.get_block(3, 5).isTransposed and not dA.get_block(3, 5).isTransposed

    def same(d, want, r=n, c=n):
        g = d.toNumpy(r, c, 1)
        assert np.array_equal(R.bits(g), R.bits(want))

    same(dA.addElement(n, n, dB, n, n, 1), a + b)       # tiled
    same(dA.addElement(n, n, dBf, n, n, 1), a + b)      # flat
    same(dA.multiplyElement(n, n, dB, n, n, 1), a * b)
    with np.errstate(divide="ignore", invalid="ignore"):
        same(dB.divideElement(n, n, dA, n, n, 1), b / a)
    same(dB.multiplyScalar(0.1), 0.1 * b)
    same(dB.addScalar(0.1), b + 0.1)
    same(dB.power(2.0), b * b)
    mat = dB.materialize()
    assert not mat.get_block(3, 5).isTransposed
    same(mat, b)
    same(dA.rowSum(n, n), R.int_sums(a).reshape(n, 1), n, 1)
    same(dA.colSum(n, n), R.int_sums(a.T).reshape(1, n), 1, n)
    same(dA.sum(n, n), R.int_sums(a.reshape(1, -1)).reshape(1, 1), 1, 1)
    same(dA.trace(n, n), np.array([[np.trace(a)]]), 1, 1)
    same(dB.project(n, n, 1, True, 123), b[123:124, :], 1, n)
    s = sess_intended
    x = rng.standard_normal(n)
    dA2 = s.fromDense(np.ascontiguousarray(b), 1)
    dv = s.fromDense(x.reshape(n, 1), 1)
    same(dA2.matrixRankOneUpdate(n, n, dv, n, 1, 1), b + np.multiply.outer(x, x))


def test_project_of_more_than_65535_blocks(sess):
    """project of row 0 of a 1 x 70000 matrix and of column 0 of a 70000 x 1 matrix at blkSize 1: the 70000 blocks of the one
    block row (column) that project reads go to extract_lines_kernel in one call, split over gridDim.y.  Bit for bit, -0.0
    included."""
    rng = np.random.default_rng(18)
    k = 70000
    v = rng.standard_normal(k) * 2.0 ** rng.integers(-30, 30, k)
    v[::7] = -0.0
    row = sess.fromDense(v.reshape(1, k), 1)
    got = row.project(1, k, 1, True, 0).toNumpy(1, k, 1)
    assert np.array_equal(R.bits(got), R.bits(v))
    col = sess.fromDense(v.reshape(k, 1), 1)
    got = col.project(k, 1, 1, False, 0).toNumpy(k, 1, 1)
    assert np.array_equal(R.bits(got), R.bits(v))


def _default_pool():
    """libcuda and device 0's default stream-ordered memory pool, which the engine allocates its result slabs from."""
    cuda = ctypes.CDLL("libcuda.so.1")
    dev, pool = ctypes.c_int(), ctypes.c_void_p()
    assert cuda.cuDeviceGet(ctypes.byref(dev), 0) == 0
    assert cuda.cuDeviceGetDefaultMemPool(ctypes.byref(pool), dev) == 0
    return cuda, pool


def pool_reserved():
    """Bytes the default pool holds from the device (CU_MEMPOOL_ATTR_RESERVED_MEM_CURRENT)."""
    cuda, pool = _default_pool()
    v = ctypes.c_uint64()
    assert cuda.cuMemPoolGetAttribute(pool, 5, ctypes.byref(v)) == 0
    return v.value


def test_sum_of_more_than_2_31_values():
    """A 46341 x 46341 block of ones (2,147,488,281 values, 17.2 GB) adopted from a torch tensor: sum, trace, rowSum, colSum and
    multiplyScalar(2).sum(), all exact.  Skipped unless 40 GiB of device memory are free.

    The engine keeps freed result slabs in the device's default pool while any session lives (mr_init raises the pool's release
    threshold), so the 17.2 GB of multiplyScalar would stay held for the rest of the process.  The test runs in a session of its
    own, hands the pool's unused memory back when that session has stopped (cuMemPoolTrimTo: another session may still be alive,
    and then mr_shutdown does not trim), frees its tensor, and checks that the pool holds no more than before the test."""
    import torch
    free, _ = torch.cuda.mem_get_info(0)
    if free < 40 * 2 ** 30:
        pytest.skip(f"needs 40 GiB of free device memory, {free / 2 ** 30:.1f} GiB free")
    n = 46341
    assert n * n == 2147488281
    t = torch.ones((n, n), dtype=torch.float64, device="cuda:0")
    torch.cuda.synchronize()
    try:
        with mb.MatfastSession(device=0) as s:
            reserved0 = pool_reserved()
            d = s.emptyDataset()
            d.put_block_device(0, 0, n, n, t.data_ptr())
            assert d.sum(n, n).get_block(0, 0).values.tolist() == [float(n * n)]
            assert d.trace(n, n).get_block(0, 0).values.tolist() == [float(n)]
            r = d.rowSum(n, n).get_block(0, 0).values
            assert r.size == n and np.all(r == n)
            c = d.colSum(n, n).get_block(0, 0).values
            assert c.size == n and np.all(c == n)
            d2 = d.multiplyScalar(2.0)
            assert d2.sum(n, n).get_block(0, 0).values.tolist() == [2.0 * n * n]
            del d2, d
            s.sync()
    finally:
        del t
        torch.cuda.empty_cache()
        cuda, pool = _default_pool()
        assert cuda.cuMemPoolTrimTo(pool, ctypes.c_size_t(0)) == 0
    assert pool_reserved() <= reserved0

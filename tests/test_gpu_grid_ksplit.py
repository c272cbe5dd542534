"""mr_dmatrix_multiply_ksplit: the grid multiply split over K (matrixMultiplyGeneral's join on k + reduceByKey(add),
MatfastExecutionHelper.scala:235-263), through ctypes, against the oracle and against the C-stationary mr_dmatrix_multiply.
Runs on the 1 x 1 grid on a one-GPU box and on every grid the box can hold (2, 4, 8 GPUs) otherwise."""
import ctypes as C

import numpy as np
import pytest

from matrel_b200 import _native as N
from oracle import matrel_oracle as O

pytestmark = pytest.mark.gpu

WORLDS = [1, 2, 4, 8]


def _ngpus():
    import torch
    return torch.cuda.device_count()


@pytest.fixture(scope="module")
def grid():
    """grid(world, algo) -> (handle, pr, pc): one single-process grid at a time, re-used across tests of the same world."""
    held = {}

    def get(world, algo=1):
        if _ngpus() < world:
            pytest.skip(f"needs {world} GPUs")
        if held.get("world") != world:
            if "g" in held:
                N.check(N.lib.mr_grid_shutdown(held.pop("g")))
            g = C.c_void_p()
            N.check(N.lib.mr_init_grid(C.byref(N.mr_options(-1, 1, algo, 0, None)), world, C.byref(g)))
            pr, pc = C.c_int32(), C.c_int32()
            N.check(N.lib.mr_grid_info(g, None, C.byref(pr), C.byref(pc), None))
            held.update(g=g, world=world, pr=pr.value, pc=pc.value)
        for r in range(world):
            ctx = C.c_void_p()
            N.check(N.lib.mr_grid_context(held["g"], r, C.byref(ctx)))
            N.check(N.lib.mr_set_option(ctx, b"gemm_algo", algo))
        return held["g"], held["pr"], held["pc"]

    yield get
    if "g" in held:
        N.check(N.lib.mr_grid_shutdown(held["g"]))


def _cdiv(a, b):
    return -(-a // b)


def _blocks(rng, n, m, blk, integer=False):
    def vals(cnt):
        return rng.integers(-8, 9, cnt).astype(np.float64) if integer else rng.uniform(-1, 1, cnt)
    return {(i, j): O.DenseMatrix(min(blk, n - i * blk), min(blk, m - j * blk), vals(min(blk, n - i * blk) * min(blk, m - j * blk)))
            for i in range(_cdiv(n, blk)) for j in range(_cdiv(m, blk))}


def _create(g, blocks, n, m, blk):
    h = C.c_void_p()
    N.check(N.lib.mr_dmatrix_create(g, n, m, blk, C.byref(h)))
    for (i, j), b in blocks.items():
        d = N.mr_block_desc()
        d.type, d.numRows, d.numCols, d.isTransposed = 1, b.numRows, b.numCols, 1 if b.isTransposed else 0
        d.values = b.values.ctypes.data_as(C.POINTER(C.c_double))
        d.valuesLen = b.values.size
        N.check(N.lib.mr_dmatrix_put_block(h, i, j, C.byref(d)))
    return h


def _block(dm, rid, cid):
    """(numRows, numCols, isTransposed, values) of a block."""
    d = N.mr_block_desc()
    N.check(N.lib.mr_dmatrix_get_block(dm, rid, cid, C.byref(d)))
    v = np.empty(d.valuesLen)
    d.values = v.ctypes.data_as(C.POINTER(C.c_double))
    N.check(N.lib.mr_dmatrix_get_block(dm, rid, cid, C.byref(d)))
    assert d.type == 1
    return d.numRows, d.numCols, bool(d.isTransposed), v


def _layout(dm, n, m, blk):
    """{(rid, cid): (numRows, numCols, isTransposed, owner, values)} of every block present."""
    out = {}
    for i in range(_cdiv(n, blk)):
        for j in range(_cdiv(m, blk)):
            has, owner = C.c_int32(), C.c_int32()
            N.check(N.lib.mr_dmatrix_has_block(dm, i, j, C.byref(has)))
            if has.value:
                N.check(N.lib.mr_dmatrix_owner(dm, i, j, C.byref(owner)))
                nr, nc, isT, v = _block(dm, i, j)
                out[(i, j)] = (nr, nc, isT, owner.value, v)
    return out


def _assemble(dm, n, m, blk):
    out = np.zeros((n, m))
    for (i, j), (nr, nc, isT, _, v) in _layout(dm, n, m, blk).items():
        assert not isT
        out[i * blk:i * blk + nr, j * blk:j * blk + nc] = v.reshape(nc, nr).T
    return out


def _num_blocks(dm):
    nb = C.c_int64()
    N.check(N.lib.mr_dmatrix_num_blocks(dm, C.byref(nb)))
    return nb.value


def _p2p(g, world):
    total = 0
    for r in range(world):
        ctx, st = C.c_void_p(), N.mr_stats()
        N.check(N.lib.mr_grid_context(g, r, C.byref(ctx)))
        N.check(N.lib.mr_get_stats(ctx, C.byref(st)))
        total += st.p2p_bytes
    return total


def _ksplit(A, B):
    out = C.c_void_p()
    N.check(N.lib.mr_dmatrix_multiply_ksplit(A, B, C.byref(out)))
    return out


def _cstat(A, B):
    out = C.c_void_p()
    N.check(N.lib.mr_dmatrix_multiply(A, B, C.byref(out)))
    return out


def _expected_p2p(world, n, k, m, blk, place_a, place_b, place_c):
    """Payload bytes the K-split moves between GPUs: rank g multiplies k-blocks [g nbk / n, (g + 1) nbk / n) and pulls the blocks of
    that range it does not own under the operand's placement; every owner reads each of its C blocks from the other contributors."""
    if world == 1:
        return 0
    nbi, nbk, nbj = _cdiv(n, blk), _cdiv(k, blk), _cdiv(m, blk)

    def ext(length, b):
        return min(blk, length - b * blk)

    def owner(place, i, j):
        return (i % place[0]) * place[1] + (j % place[1])

    contributors = [r for r in range(world) if nbk * (r + 1) // world > nbk * r // world]
    total = 0
    for r in contributors:
        for kk in range(nbk * r // world, nbk * (r + 1) // world):
            total += sum(ext(n, i) * ext(k, kk) for i in range(nbi) if owner(place_a, i, kk) != r)
            total += sum(ext(k, kk) * ext(m, j) for j in range(nbj) if owner(place_b, kk, j) != r)
    for i in range(nbi):
        for j in range(nbj):
            total += ext(n, i) * ext(m, j) * (len(contributors) - (owner(place_c, i, j) in contributors))
    return 8 * total


def _operands(g, rng, case, integer=False):
    """(A, B, oracle A, oracle B, n, k, m, blk, handles to free).  "gram" cases: A = X^T through mr_dmatrix_transpose (row-major
    blocks, flag-transposed slabs) and B = X, X = rows x cols."""
    kind, blk = case[0], case[-1]
    if kind == "gram":
        rows, cols = case[1], case[2]
        Xo = _blocks(rng, rows, cols, blk, integer)
        X, At = _create(g, Xo, rows, cols, blk), C.c_void_p()
        N.check(N.lib.mr_dmatrix_transpose(X, C.byref(At)))
        return At, X, O.transpose(Xo), Xo, cols, rows, cols, blk, [X, At]
    n, k, m = case[1], case[2], case[3]
    Ao, Bo = _blocks(rng, n, k, blk, integer), _blocks(rng, k, m, blk, integer)
    A, B = _create(g, Ao, n, k, blk), _create(g, Bo, k, m, blk)
    return A, B, Ao, Bo, n, k, m, blk, [A, B]


CASES = {
    "gram": ("gram", 2555, 121, 64),          # tall-skinny X^T X: 40 k-blocks, C 2 x 2
    "single": ("gram", 2555, 50, 64),         # W^T W: one output block
    "k3": ("plain", 300, 3 * 64 - 5, 260, 64),  # fewer k-blocks than GPUs
    "k1": ("plain", 200, 40, 150, 64),        # one k-block: the outer-product branch
    "square": ("plain", 7 * 64 - 6, 5 * 64, 6 * 64 - 10, 64),
    "odd": ("plain", 4 * 45 - 7, 9 * 45 - 2, 3 * 45 + 4, 45),  # slots start on 8-byte boundaries: the kernel's scalar path
}


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("algo", [1, 4])
@pytest.mark.parametrize("world", WORLDS)
def test_ksplit_matches_oracle(grid, world, algo, case):
    """Values against the oracle, the C-stationary layout (ids, shapes, owners, block count) and the bytes moved between GPUs."""
    g, pr, pc = grid(world, algo)
    rng = np.random.default_rng([world, algo, len(case), ord(case[0])])
    A, B, Ao, Bo, n, k, m, blk, free = _operands(g, rng, CASES[case])
    before = _p2p(g, world)
    Ck = _ksplit(A, B)
    moved = _p2p(g, world) - before
    Cs = _cstat(A, B)
    want = O.assemble(O.matrix_multiply(Ao, n, k, Bo, k, m, blk), n, m, blk)
    got = _assemble(Ck, n, m, blk)
    assert np.max(np.abs(got - want)) <= 1e-12 * np.max(np.abs(want))
    assert _num_blocks(Ck) == _num_blocks(Cs) == _cdiv(n, blk) * _cdiv(m, blk)
    lk, ls = _layout(Ck, n, m, blk), _layout(Cs, n, m, blk)
    assert {key: v[:4] for key, v in lk.items()} == {key: v[:4] for key, v in ls.items()}
    assert all(v[3] == (i % pr) * pc + (j % pc) for (i, j), v in lk.items())
    assert moved == _expected_p2p(world, n, k, m, blk, (pr, pc), (pr, pc), (pr, pc))
    for h in free + [Ck, Cs]:
        N.check(N.lib.mr_dmatrix_free(h))


@pytest.mark.parametrize("case", ["gram", "square", "odd"])
@pytest.mark.parametrize("algo", [1, 4])
@pytest.mark.parametrize("world", WORLDS)
def test_ksplit_bit_identical_to_c_stationary_on_integers(grid, world, algo, case):
    """Small-integer operands: every partial and every sum is exact in fp64, so the K-split and the C-stationary multiply agree in
    every bit, whatever the order of the additions."""
    g, _, _ = grid(world, algo)
    rng = np.random.default_rng([world, algo, 7, ord(case[0])])
    A, B, _, _, n, _, m, blk, free = _operands(g, rng, CASES[case], integer=True)
    Ck, Cs = _ksplit(A, B), _cstat(A, B)
    lk, ls = _layout(Ck, n, m, blk), _layout(Cs, n, m, blk)
    assert lk.keys() == ls.keys() and _num_blocks(Ck) == _num_blocks(Cs)
    for key in lk:
        assert lk[key][:4] == ls[key][:4]
        assert np.array_equal(lk[key][4], ls[key][4]), key
    for h in free + [Ck, Cs]:
        N.check(N.lib.mr_dmatrix_free(h))


@pytest.mark.parametrize("algo", [1, 4])
@pytest.mark.parametrize("world", WORLDS)
def test_ksplit_is_deterministic(grid, world, algo):
    """Two runs on the same U(-1, 1) operands agree bitwise (fixed summation order); on one GPU it is the ordinary multiply."""
    g, _, _ = grid(world, algo)
    rng = np.random.default_rng([world, algo, 11])
    A, B, _, _, n, _, m, blk, free = _operands(g, rng, CASES["gram"])
    C1, C2 = _ksplit(A, B), _ksplit(A, B)
    r1 = _assemble(C1, n, m, blk)
    assert np.array_equal(r1, _assemble(C2, n, m, blk))
    handles = [C1, C2]
    if world == 1:
        Cs = _cstat(A, B)
        assert np.array_equal(r1, _assemble(Cs, n, m, blk))
        handles.append(Cs)
    for h in free + handles:
        N.check(N.lib.mr_dmatrix_free(h))


@pytest.mark.parametrize("world", WORLDS)
def test_ksplit_accepts_operands_on_other_placements(grid, world):
    """B re-partitioned to the column layout (1, world) and A flag-transposed are used where they are (no re-partitioning: the
    bytes moved follow the operands' own placements); the result is the same and feeds the other grid operators."""
    g, pr, pc = grid(world, 1)
    rows, cols, blk = 1500, 130, 64
    rng = np.random.default_rng(world + 31)
    Xo, Yo = _blocks(rng, rows, cols, blk), _blocks(rng, rows, 2 * cols, blk)
    X, Y = _create(g, Xo, rows, cols, blk), _create(g, Yo, rows, 2 * cols, blk)
    Xt, Yc = C.c_void_p(), C.c_void_p()
    N.check(N.lib.mr_dmatrix_transpose(X, C.byref(Xt)))
    N.check(N.lib.mr_dmatrix_repartition(Y, 1, world, C.byref(Yc)))
    before = _p2p(g, world)
    Cp = _ksplit(Xt, Yc)                   # X^T Y with Y on (1, world)
    moved = _p2p(g, world) - before
    Cg = _ksplit(Xt, Y)                    # the same with Y on the grid's placement
    n, k, m = cols, rows, 2 * cols
    got = _assemble(Cp, n, m, blk)
    assert np.array_equal(got, _assemble(Cg, n, m, blk))
    want = O.assemble(O.matrix_multiply(O.transpose(Xo), n, k, Yo, k, m, blk), n, m, blk)
    assert np.max(np.abs(got - want)) <= 1e-12 * np.max(np.abs(want))
    assert moved == _expected_p2p(world, n, k, m, blk, (pr, pc), (1, world), (pr, pc))
    S, total = C.c_void_p(), C.c_double()
    N.check(N.lib.mr_dmatrix_elementwise(0, Cp, Cg, C.byref(S)))
    assert np.array_equal(_assemble(S, n, m, blk), got + got)
    N.check(N.lib.mr_dmatrix_reduce_scalar(Cp, 0, C.byref(total)))
    assert abs(total.value - want.sum()) <= 1e-10 * np.abs(want).sum()
    for h in (X, Y, Xt, Yc, Cp, Cg, S):
        N.check(N.lib.mr_dmatrix_free(h))


@pytest.mark.parametrize("world", WORLDS)
def test_ksplit_errors(grid, world):
    """The argument checks of mr_dmatrix_multiply, as status returns."""
    g, _, _ = grid(world, 1)
    A, B, out = C.c_void_p(), C.c_void_p(), C.c_void_p()
    N.check(N.lib.mr_dmatrix_rand(g, 200, 130, 64, 1, C.byref(A)))
    N.check(N.lib.mr_dmatrix_rand(g, 120, 90, 64, 2, C.byref(B)))
    assert N.lib.mr_dmatrix_multiply_ksplit(A, B, C.byref(out)) == N.MR_EDIM
    assert "Matrix dimension not match, leftColNum = 130, rightRowNum = 120" in N.last_error()
    assert N.lib.mr_dmatrix_multiply_ksplit(A, None, C.byref(out)) == N.MR_EINVAL
    B32 = C.c_void_p()
    N.check(N.lib.mr_dmatrix_rand(g, 130, 90, 32, 3, C.byref(B32)))
    assert N.lib.mr_dmatrix_multiply_ksplit(A, B32, C.byref(out)) == N.MR_EINVAL
    g2, B2 = C.c_void_p(), C.c_void_p()
    N.check(N.lib.mr_init_grid(C.byref(N.mr_options(-1, 1, 1, 0, None)), world, C.byref(g2)))
    try:
        N.check(N.lib.mr_dmatrix_rand(g2, 130, 90, 64, 4, C.byref(B2)))
        assert N.lib.mr_dmatrix_multiply_ksplit(A, B2, C.byref(out)) == N.MR_EINVAL
        assert "different grids" in N.last_error()
        N.check(N.lib.mr_dmatrix_free(B2))
    finally:
        N.check(N.lib.mr_grid_shutdown(g2))
    for h in (A, B, B32):
        N.check(N.lib.mr_dmatrix_free(h))

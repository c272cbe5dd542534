"""Host-resident datasets and the streamed multiply.

The streamed product (a host-resident operand, C computed tile by tile through the device) must be BIT-IDENTICAL to the
resident one: same block ids, formats, flags and values, for gemm_algo 0 (both engines), 1 and 4, every shape and storage format.  Every case runs
under the smallest power-of-two `stream_budget_mb` that fits, so it really tiles (asserted through `stream_tiles`).  Around
that: the loop order that moves fewer bytes, the per-tile fallback of the Ozaki-II engine on NaN, the errors, the round trip
between residences, and one product at N = 32768."""
import numpy as np
import pytest

import matrel_b200 as mb
from tests.exact_ref import alpha_of, fp64_dot_bound, moduli_for, oz2_bound

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------------------------------
# fixtures of this file
# ---------------------------------------------------------------------------------------------------------------------------
def _dense_blocks(M, N, blk, rng, transposed=lambda i, j: False, absent=()):
    out = {}
    for i in range(-(-M // blk)):
        for j in range(-(-N // blk)):
            if (i, j) in absent:
                continue
            a = rng.uniform(-1, 1, (min(blk, M - i * blk), min(blk, N - j * blk)))
            out[(i, j)] = mb.DenseMatrix.from_numpy(a, transposed_storage=transposed(i, j))
    return out


def _sparse(a, csr):
    """CSC (or CSR) SparseMatrix of the dense array a."""
    if csr:
        t = _sparse(a.T, False)
        return mb.SparseMatrix(a.shape[0], a.shape[1], t.colPtrs, t.rowIndices, t.values, True)
    ptr, idx, val = [0], [], []
    for c in range(a.shape[1]):
        nz = np.nonzero(a[:, c])[0]
        idx.extend(nz.tolist())
        val.extend(a[nz, c].tolist())
        ptr.append(len(idx))
    return mb.SparseMatrix(a.shape[0], a.shape[1], ptr, idx, val, False)


def _sparse_blocks(M, N, blk, rng, density, csr=lambda i, j: False):
    out = {}
    for i in range(-(-M // blk)):
        for j in range(-(-N // blk)):
            r, c = min(blk, M - i * blk), min(blk, N - j * blk)
            a = np.where(rng.uniform(0, 1, (r, c)) < density, rng.uniform(-1, 1, (r, c)), 0.0)
            out[(i, j)] = _sparse(a, csr(i, j))
    return out


def _load(s, blocks, host):
    rows = [mb.MatrixBlock(i, j, m) for (i, j), m in sorted(blocks.items())]
    return s.createHostDataset(rows) if host else s.createDataset(rows)


def _dump(ds):
    """{(rid, cid): (kind, isT, rows, cols, values as int64 bits, colPtrs, rowIndices)}: equal dumps = bit-identical datasets."""
    out = {}
    for b in ds.collect():
        m = b.matrix
        sp = isinstance(m, mb.SparseMatrix)
        out[(b.rid, b.cid)] = ("sparse" if sp else "dense", m.isTransposed, m.numRows, m.numCols, m.values.view(np.int64).copy(),
                               m.colPtrs.copy() if sp else None, m.rowIndices.copy() if sp else None)
    return out


def _assert_identical(got, want):
    assert sorted(got) == sorted(want)
    for k in want:
        g, w = got[k], want[k]
        assert g[:4] == w[:4], (k, g[:4], w[:4])
        assert np.array_equal(g[4], w[4]), f"block {k}: values differ"
        for x, y in ((g[5], w[5]), (g[6], w[6])):
            assert (x is None) == (y is None) and (x is None or np.array_equal(x, y)), f"block {k}: index arrays differ"


def _assemble(ds, M, N, blk):
    out = np.zeros((M, N))
    for b in ds.collect():
        out[b.rid * blk:b.rid * blk + b.matrix.numRows, b.cid * blk:b.cid * blk + b.matrix.numCols] = b.matrix.to_numpy()
    return out


def _streamed(s, A, B, M, K, N, blk, budgets_mb=(1, 2, 4, 8, 16, 32, 64, 128, 256, 512, 1024, 2048, 4096)):
    """A x B under the smallest budget of `budgets_mb` that fits; returns (C, stats)."""
    for mbytes in budgets_mb:
        s.set_option("stream_budget_mb", mbytes)
        s.reset_stats()
        try:
            C = A.matrixMultiply(M, K, B, K, N, blk)
        except MemoryError:
            continue
        s.sync()
        st = s.stats()
        s.set_option("stream_budget_mb", 0)
        return C, st
    raise AssertionError("no budget fits")


def _host_bytes(blocks):
    return sum(m.values.size * 8 + (m.colPtrs.size * 4 + m.rowIndices.size * 4 if isinstance(m, mb.SparseMatrix) else 0)
               for m in blocks.values())


def _check_bit_identical(algo, Ab, Bb, M, K, N, blk, residence="AB", min_tiles=4):
    with mb.MatfastSession(device=0, gemm_algo=algo) as s:
        want = _dump(_load(s, Ab, False).matrixMultiply(M, K, _load(s, Bb, False), K, N, blk))
        A, B = _load(s, Ab, "A" in residence), _load(s, Bb, "B" in residence)
        C, st = _streamed(s, A, B, M, K, N, blk)
        assert C.isHost
        assert st["stream_tiles"] >= min_tiles, st["stream_tiles"]
        _assert_identical(_dump(C), want)
        return st


# ---------------------------------------------------------------------------------------------------------------------------
# bit-identity, streamed against resident
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("residence", ["A", "B", "AB"])
def test_auto_above_the_engine_threshold(residence):
    """2 M K N >= 2^33: the whole product takes the Ozaki-II engine, and so must every tile (a 1 x 1 tile alone is below it)."""
    rng = np.random.default_rng(1)
    M, K, N, blk = 2000, 2100, 1900, 512
    _check_bit_identical(0, _dense_blocks(M, K, blk, rng), _dense_blocks(K, N, blk, rng), M, K, N, blk, residence)


def test_auto_below_the_engine_threshold():
    rng = np.random.default_rng(2)
    M, K, N, blk = 1000, 1100, 900, 256
    _check_bit_identical(0, _dense_blocks(M, K, blk, rng), _dense_blocks(K, N, blk, rng), M, K, N, blk)


@pytest.mark.parametrize("algo", [1, 4])
def test_forced_engines(algo):
    rng = np.random.default_rng(3 + algo)
    M, K, N, blk = 1500, 1300, 1700, 384
    _check_bit_identical(algo, _dense_blocks(M, K, blk, rng), _dense_blocks(K, N, blk, rng), M, K, N, blk)


@pytest.mark.parametrize("algo", [0, 1])
def test_ragged_absent_and_transposed_blocks(algo):
    """blk divides none of M, K, N; some blocks of both operands are absent; row-major and column-major blocks mixed."""
    rng = np.random.default_rng(5)
    M, K, N, blk = 2300, 2050, 2200, 500
    Ab = _dense_blocks(M, K, blk, rng, transposed=lambda i, j: (i + j) % 2 == 0, absent={(1, 2), (3, 0)})
    Bb = _dense_blocks(K, N, blk, rng, transposed=lambda i, j: (i * j) % 3 == 1, absent={(0, 4), (2, 2)})
    _check_bit_identical(algo, Ab, Bb, M, K, N, blk)


# A CSC LEFT block is multiplied by a scatter kernel whose adds are atomic (spmm_csc_kernel): its sums are not reproducible from
# one run to the next even without streaming, so CSC left operands are held to the resident result within rounding (below), and
# the bit-identity cases take CSR left blocks and CSC / CSR right blocks.
@pytest.mark.parametrize("residence", ["A", "B", "AB"])
def test_sparse_times_dense(residence):
    """CSR left blocks (density 0.05 -> the fused sparse x dense kernels) against dense B."""
    rng = np.random.default_rng(6)
    M, K, N, blk = 1024, 1024, 768, 256
    Ab = _sparse_blocks(M, K, blk, rng, 0.05, csr=lambda i, j: True)
    _check_bit_identical(0, Ab, _dense_blocks(K, N, blk, rng), M, K, N, blk, residence)


@pytest.mark.parametrize("algo", [0, 1])
def test_dense_times_csc_and_csr(algo):
    """Sparse RIGHT blocks (CSC and CSR) are densified into the dense GEMM."""
    rng = np.random.default_rng(16)
    M, K, N, blk = 1024, 768, 1024, 256
    Bb = _sparse_blocks(K, N, blk, rng, 0.05, csr=lambda i, j: (i + j) % 2 == 1)
    _check_bit_identical(algo, _dense_blocks(M, K, blk, rng), Bb, M, K, N, blk)


def test_sparse_times_sparse_keeps_sparse_outputs():
    """Low-density sparse x sparse: the output blocks replay the reference's format chains, and stay sparse."""
    rng = np.random.default_rng(7)
    M, K, N, blk = 1024, 768, 1024, 256
    Ab = _sparse_blocks(M, K, blk, rng, 0.004, csr=lambda i, j: True)
    Bb = _sparse_blocks(K, N, blk, rng, 0.004, csr=lambda i, j: j % 2 == 1)
    with mb.MatfastSession(device=0) as s:
        want = _dump(_load(s, Ab, False).matrixMultiply(M, K, _load(s, Bb, False), K, N, blk))
        assert any(v[0] == "sparse" for v in want.values())
        C, st = _streamed(s, _load(s, Ab, True), _load(s, Bb, True), M, K, N, blk, budgets_mb=(1, 2, 4, 8, 16))
        assert st["stream_tiles"] >= 4
        _assert_identical(_dump(C), want)


@pytest.mark.parametrize("density", [0.05, 0.004])
def test_csc_left_operands_match_within_rounding(density):
    """CSC left blocks x dense (0.05) and x CSC / CSR (0.004, the format chains): the same ids, formats, flags and index arrays
    as the resident product; values within a few units of rounding of it."""
    rng = np.random.default_rng(17)
    M, K, N, blk = 1024, 768, 1024, 256
    Ab = _sparse_blocks(M, K, blk, rng, density)
    Bb = _dense_blocks(K, N, blk, rng) if density > 0.01 else _sparse_blocks(K, N, blk, rng, density, csr=lambda i, j: j % 2 == 1)
    with mb.MatfastSession(device=0) as s:
        R = _load(s, Ab, False).matrixMultiply(M, K, _load(s, Bb, False), K, N, blk)
        want = _dump(R)
        C, st = _streamed(s, _load(s, Ab, True), _load(s, Bb, True), M, K, N, blk, budgets_mb=(1, 2, 4, 8, 16))
        assert st["stream_tiles"] >= 4
        got = _dump(C)
        assert sorted(got) == sorted(want)
        for k in want:
            assert got[k][:4] == want[k][:4]
            for x, y in ((got[k][5], want[k][5]), (got[k][6], want[k][6])):
                assert (x is None) == (y is None) and (x is None or np.array_equal(x, y)), k
        assert np.allclose(_assemble(C, M, N, blk), _assemble(R, M, N, blk), rtol=1e-14, atol=1e-14)


# ---------------------------------------------------------------------------------------------------------------------------
# the loop order and the traffic
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("larger", ["A", "B"])
def test_outer_operand_moves_each_operand_once(larger):
    """One block row of A (or one block column of B): taking that operand as the outer panel moves every byte once,
    |A| + |B|; the other order would move the small operand once per tile.  d2h = |C|."""
    rng = np.random.default_rng(8)
    blk = 256
    M, K, N = (4096, 1024, 256) if larger == "A" else (256, 1024, 4096)
    Ab, Bb = _dense_blocks(M, K, blk, rng), _dense_blocks(K, N, blk, rng)
    with mb.MatfastSession(device=0, gemm_algo=1) as s:
        C, st = _streamed(s, _load(s, Ab, True), _load(s, Bb, True), M, K, N, blk)
        assert st["stream_tiles"] >= 2
        assert st["stream_h2d_bytes"] == _host_bytes(Ab) + _host_bytes(Bb), (st["stream_h2d_bytes"], _host_bytes(Ab), _host_bytes(Bb))
        assert st["stream_d2h_bytes"] == M * N * 8
        # the library-wide counters also carry the tiles' descriptor tables
        assert st["h2d_bytes"] > st["stream_h2d_bytes"] and st["d2h_bytes"] >= st["stream_d2h_bytes"]


def test_h2d_bytes_follow_the_tiling_formula():
    """Square operands: |outer| + (outer panels) |inner|, whichever order."""
    rng = np.random.default_rng(9)
    M = K = N = 1536
    blk = 256
    Ab, Bb = _dense_blocks(M, K, blk, rng), _dense_blocks(K, N, blk, rng)
    with mb.MatfastSession(device=0, gemm_algo=1) as s:
        C, st = _streamed(s, _load(s, Ab, True), _load(s, Bb, True), M, K, N, blk)
        a, b = _host_bytes(Ab), _host_bytes(Bb)
        assert st["stream_tiles"] >= 4
        moved = st["stream_h2d_bytes"]
        assert any(moved == a + p * b or moved == b + p * a for p in range(2, 7)), moved


# ---------------------------------------------------------------------------------------------------------------------------
# the Ozaki-II fallback is per tile
# ---------------------------------------------------------------------------------------------------------------------------
def test_nan_in_one_block_row_falls_back_per_tile():
    rng = np.random.default_rng(10)
    M, K, N, blk = 2048, 2048, 2048, 512
    Ab, Bb = _dense_blocks(M, K, blk, rng), _dense_blocks(K, N, blk, rng)
    a = Ab[(1, 2)].to_numpy().copy()
    a[7, 11] = np.nan
    Ab[(1, 2)] = mb.DenseMatrix.from_numpy(a)
    with mb.MatfastSession(device=0) as s:
        resident = _assemble(_load(s, Ab, False).matrixMultiply(M, K, _load(s, Bb, False), K, N, blk), M, N, blk)
        C, st = _streamed(s, _load(s, Ab, True), _load(s, Bb, True), M, K, N, blk)
        assert st["stream_tiles"] >= 4
        got = _assemble(C, M, N, blk)
    assert np.array_equal(np.isnan(got), np.isnan(resident))
    Ad = np.vstack([np.hstack([Ab[(i, k)].to_numpy() for k in range(4)]) for i in range(4)])
    Bd = np.vstack([np.hstack([Bb[(k, j)].to_numpy() for j in range(4)]) for k in range(4)])
    ok = ~np.isnan(Ad).any(axis=1)
    ref = Ad[ok] @ Bd
    bound = oz2_bound(Ad[ok], Bd, alpha_of(moduli_for(K), K), ref) + fp64_dot_bound(Ad[ok], Bd)  # Ozaki-II or exact-kernel tiles
    assert np.all(np.abs(got[ok] - ref) <= bound)
    assert np.all(np.isnan(got[~ok]))


# ---------------------------------------------------------------------------------------------------------------------------
# errors
# ---------------------------------------------------------------------------------------------------------------------------
def test_budget_below_one_block_row_and_column():
    rng = np.random.default_rng(11)
    M = K = N = 1024
    blk = 512
    with mb.MatfastSession(device=0) as s:
        A, B = _load(s, _dense_blocks(M, K, blk, rng), True), _load(s, _dense_blocks(K, N, blk, rng), True)
        s.set_option("stream_budget_mb", 1)
        with pytest.raises(MemoryError, match=r"one block row x one block column with full K needs \d+ bytes .* budget is 1048576 bytes"):
            A.matrixMultiply(M, K, B, K, N, blk)


def _other_operators(d, v, n, blk):
    return {
        "mr_transpose": lambda: d.transpose(),
        "mr_add_element": lambda: d.addElement(n, n, d, n, n, blk),
        "mr_multiply_element": lambda: d.multiplyElement(n, n, d, n, n, blk),
        "mr_divide_element": lambda: d.divideElement(n, n, d, n, n, blk),
        "mr_add_scalar": lambda: d.addScalar(1.0),
        "mr_multiply_scalar": lambda: d.multiplyScalar(2.0),
        "mr_power": lambda: d.power(2.0),
        "mr_rank_one_update": lambda: d.matrixRankOneUpdate(n, n, v, n, 1, blk),
        "mr_materialize": lambda: d.materialize(),
        "mr_row_sum": lambda: d.rowSum(n, n),
        "mr_col_sum": lambda: d.colSum(n, n),
        "mr_sum": lambda: d.sum(n, n),
        "mr_trace": lambda: d.trace(n, n),
        "mr_project": lambda: d.project(n, n, blk, True, 3),
        "mr_selection": lambda: d.selection(n, n, blk, 3, 4),
        "mr_vec": lambda: d.vec(n, n, blk),
        "mr_matrix_filter_blocks": lambda: d.filter_blocks(2, 0, 1, 0),
    }


def test_other_operators_refuse_host_datasets_and_run_after_to_device():
    rng = np.random.default_rng(12)
    n, blk = 96, 48
    with mb.MatfastSession(device=0, compat_bugs=False) as s:
        hd = _load(s, _dense_blocks(n, n, blk, rng), True)
        hv = _load(s, _dense_blocks(n, 1, blk, rng), True)
        for name, op in _other_operators(hd, hv.toDevice(), n, blk).items():
            with pytest.raises(mb.UnsupportedOperation, match=f"{name}: .*mr_matrix_to_device"):
                op()
        with pytest.raises(mb.UnsupportedOperation, match="mr_matrix_to_device"):
            hd.block_device_ptr(0, 0)
        dd, dv = hd.toDevice(), hv.toDevice()
        assert not dd.isHost and hd.isHost
        for name, op in _other_operators(dd, dv, n, blk).items():
            assert op() is not None, name
        s.sync()


# ---------------------------------------------------------------------------------------------------------------------------
# round trip between the residences
# ---------------------------------------------------------------------------------------------------------------------------
def test_round_trip_and_put_copies_the_callers_arrays():
    rng = np.random.default_rng(13)
    blocks = _dense_blocks(300, 200, 128, rng, transposed=lambda i, j: j == 1)
    blocks.update({(i + 5, j): m for (i, j), m in _sparse_blocks(256, 256, 128, rng, 0.05, csr=lambda i, j: i == j).items()})
    want = {k: (type(m).__name__, m.isTransposed, m.values.copy()) for k, m in blocks.items()}
    with mb.MatfastSession(device=0) as s:
        h = _load(s, blocks, True)
        for m in blocks.values():      # the caller's arrays are free once put_block has returned
            m.values[:] = -7.0
        assert h.isHost and sorted(h.block_ids()) == sorted(blocks)
        for k, (kind, isT, vals) in want.items():
            got = h.get_block(*k)
            assert (type(got).__name__, got.isTransposed) == (kind, isT)
            assert np.array_equal(got.values, vals)
        d = h.toDevice()
        assert not d.isHost
        back = d.toHost()
        assert back.isHost
        _assert_identical(_dump(back), _dump(h))
        _assert_identical(_dump(d), _dump(h))


def test_to_host_copies_before_the_source_is_released():
    """The device source of toHost() may be freed right after the call while its copies still run on the egress stream: the
    release must wait for them, or the next allocation (here another generator of the same size) overwrites the blocks first."""
    n, blk = 8192, 1024
    with mb.MatfastSession(device=0) as s:
        h = s.rand(n, n, blk, 42).toHost()     # the device dataset is dropped at once
        other = s.rand(n, n, blk, 43)           # reuses its memory from the pool
        ref = s.rand(n, n, blk, 42)
        s.sync()
        for rid, cid in ref.block_ids():
            assert np.array_equal(h.get_block(rid, cid).values.view(np.int64), ref.get_block(rid, cid).values.view(np.int64)), (rid, cid)
        del other


def test_streamed_result_feeds_another_streamed_multiply():
    """The write-back of one streamed product is read by the next one (its blocks' events order the copies)."""
    rng = np.random.default_rng(14)
    n, blk = 1024, 256
    Ab, Bb = _dense_blocks(n, n, blk, rng), _dense_blocks(n, n, blk, rng)
    with mb.MatfastSession(device=0, gemm_algo=1) as s:
        dA, dB = _load(s, Ab, False), _load(s, Bb, False)
        want = _dump(dA.matrixMultiply(n, n, dB, n, n, blk).matrixMultiply(n, n, dB, n, n, blk))
        s.set_option("stream_budget_mb", 8)
        C1 = _load(s, Ab, True).matrixMultiply(n, n, _load(s, Bb, True), n, n, blk)
        C2 = C1.matrixMultiply(n, n, dB, n, n, blk)
        assert C2.isHost and s.stats()["stream_tiles"] >= 4
        _assert_identical(_dump(C2), want)


# ---------------------------------------------------------------------------------------------------------------------------
# at size
# ---------------------------------------------------------------------------------------------------------------------------
def _mem_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def test_at_size_freivalds_and_bit_identity():
    import torch
    n, blk = 32768, 2048
    free, _ = torch.cuda.mem_get_info(0)
    if free < 3 * n * n * 8 + (18 << 30):
        pytest.skip(f"needs {(3 * n * n * 8 + (18 << 30)) >> 30} GiB of device memory for the resident reference")
    if _mem_available() < 3 * n * n * 8 + (16 << 30):
        pytest.skip(f"needs {(3 * n * n * 8 + (16 << 30)) >> 30} GiB of available host memory")
    rng = np.random.default_rng(15)
    with mb.MatfastSession(device=0) as s:
        A, B = s.rand(n, n, blk, 42), s.rand(n, n, blk, 43)
        resident = A.matrixMultiply(n, n, B, n, n, blk)
        hA, hB = A.toHost(), B.toHost()
        C, st = _streamed(s, hA, hB, n, n, n, blk, budgets_mb=tuple(range(2048, 40960, 2048)))
        assert st["stream_tiles"] >= 4, st["stream_tiles"]
        for rid, cid in resident.block_ids():
            assert np.array_equal(C.get_block(rid, cid).values.view(np.int64), resident.get_block(rid, cid).values.view(np.int64))
        assert sorted(C.block_ids()) == sorted(resident.block_ids())
        del resident, hA, hB
        # Freivalds over every block: C x = A (B x), with the exact kernel for the mat-vecs
        s.set_option("gemm_algo", 1)
        Cd = C.toDevice()
        x = rng.uniform(-1, 1, n)
        dx = s.createDataset(mb.MatrixBlock(i, 0, mb.DenseMatrix(blk, 1, x[i * blk:(i + 1) * blk].copy())) for i in range(n // blk))
        vec = lambda ds: _assemble(ds, n, 1, blk)[:, 0]
        ABx = vec(A.matrixMultiply(n, n, B.matrixMultiply(n, n, dx, n, 1, blk), n, 1, blk))
        Cx = vec(Cd.matrixMultiply(n, n, dx, n, 1, blk))
        assert np.max(np.abs(Cx - ABx) / (np.abs(ABx) + n * 1e-3)) <= 1e-11

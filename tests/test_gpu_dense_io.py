"""Whole dense matrices in and out of datasets: MatfastSession.fromDense, Dataset.toNumpy / Dataset.toTorch (mr_matrix_from_dense /
mr_matrix_to_dense).  Ingest and assembly only copy, so every comparison is exact: round trips, the blocks fromDense makes, a
product of such datasets against one of datasets built block by block, and the assembly of arbitrary datasets (mixed layouts,
CSC / CSR blocks, absent and ragged blocks, host-resident and streamed results) against a numpy assembly of collect()."""
import ctypes as C

import numpy as np
import pytest
import torch

import matrel_b200 as mb
from matrel_b200 import _native as N

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sess():
    with mb.MatfastSession(device=0) as s:
        yield s


def _assemble(ds, M, N, blk):
    out = np.zeros((M, N))
    for b in ds.collect():
        out[b.rid * blk:b.rid * blk + b.matrix.numRows, b.cid * blk:b.cid * blk + b.matrix.numCols] = b.matrix.to_numpy()
    return out


def _dump(ds):
    """{(rid, cid): (kind, isT, rows, cols, values as int64 bits)}: equal dumps = bit-identical dense datasets."""
    return {(b.rid, b.cid): (type(b.matrix).__name__, b.matrix.isTransposed, b.matrix.numRows, b.matrix.numCols,
                             b.matrix.values.view(np.int64).tobytes()) for b in ds.collect()}


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


def _check_all_out(ds, A, blk):
    """toNumpy (both orders) and toTorch give A exactly."""
    M, Nc = A.shape
    for order in ("C", "F"):
        got = ds.toNumpy(M, Nc, blk, order=order)
        assert got.flags[order + "_CONTIGUOUS"]
        assert np.array_equal(got, A), order
    t = ds.toTorch(M, Nc, blk)
    assert t.is_cuda and t.is_contiguous() and t.dtype == torch.float64 and tuple(t.shape) == (M, Nc)
    assert np.array_equal(t.cpu().numpy(), A)


SHAPES = [(300, 200, 64), (50, 70, 128), (1, 257, 32), (257, 1, 32), (256, 192, 64)]
SOURCES = ["C", "F", "C_slice", "F_slice", "pinned", "cuda", "cuda_slice", "cuda_colmajor"]


def _source(kind, A):
    """(the object passed to fromDense, whether it is row-major)"""
    M, Nc = A.shape
    if kind == "C":
        return np.ascontiguousarray(A), True
    if kind == "F":
        return np.asfortranarray(A), False
    if kind == "C_slice":  # ld > ncols and a base that is only 8-byte aligned
        big = np.full((M + 5, Nc + 7), np.nan)
        big[2:2 + M, 3:3 + Nc] = A
        return big[2:2 + M, 3:3 + Nc], True
    if kind == "F_slice":
        big = np.asfortranarray(np.full((M + 3, Nc + 4), np.nan))
        big[1:1 + M, 2:2 + Nc] = A
        return big[1:1 + M, 2:2 + Nc], False
    if kind == "pinned":
        return torch.from_numpy(np.ascontiguousarray(A)).pin_memory(), True
    if kind == "cuda":
        return torch.from_numpy(np.ascontiguousarray(A)).cuda(), True
    if kind == "cuda_slice":
        big = torch.full((M + 3, Nc + 5), float("nan"), dtype=torch.float64, device="cuda")
        big[1:1 + M, 1:1 + Nc] = torch.from_numpy(A)
        return big[1:1 + M, 1:1 + Nc], True
    if kind == "cuda_colmajor":  # a transposed view: unit stride down the columns
        return torch.from_numpy(np.ascontiguousarray(A.T)).cuda().T, False
    raise AssertionError(kind)


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("kind", SOURCES)
def test_round_trip_is_exact(sess, shape, kind):
    M, Nc, blk = shape
    A = np.random.default_rng(M * 7 + Nc).uniform(-1, 1, (M, Nc))
    src, rm = _source(kind, A)
    ds = sess.fromDense(src, blk)
    assert not ds.isHost
    nbr, nbc = -(-M // blk), -(-Nc // blk)
    assert ds.block_ids() == [(i, j) for i in range(nbr) for j in range(nbc)]
    if M == 1 or Nc == 1:  # a single line is contiguous both ways: the flag only has to be the same on every block
        rm = ds.collect()[0].matrix.isTransposed
    for b in ds.collect():
        assert isinstance(b.matrix, mb.DenseMatrix) and b.matrix.isTransposed == rm
        assert (b.matrix.numRows, b.matrix.numCols) == (min(blk, M - b.rid * blk), min(blk, Nc - b.cid * blk))
    assert np.array_equal(_assemble(ds, M, Nc, blk), A)
    _check_all_out(ds, A, blk)


@pytest.mark.parametrize("kind", ["C", "F_slice", "pinned", "cuda_slice"])
def test_host_resident_target(sess, kind):
    M, Nc, blk = 300, 200, 64
    A = np.random.default_rng(5).uniform(-1, 1, (M, Nc))
    src, rm = _source(kind, A)
    ds = sess.fromDense(src, blk, host=True)
    assert ds.isHost
    assert all(b.matrix.isTransposed == rm for b in ds.collect())
    assert np.array_equal(_assemble(ds, M, Nc, blk), A)
    _check_all_out(ds, A, blk)
    assert np.array_equal(_assemble(ds.toDevice(), M, Nc, blk), A)


def test_ingest_and_egress_bytes_are_counted(sess):
    M, Nc, blk = 300, 200, 64
    A = np.random.default_rng(6).uniform(-1, 1, (M, Nc))
    sess.sync()
    sess.reset_stats()
    ds = sess.fromDense(A, blk)
    st = sess.stats()
    assert st["h2d_bytes"] == M * Nc * 8 and st["kernel_launches"] == 0
    sess.reset_stats()
    ds.toNumpy(M, Nc, blk)
    st = sess.stats()
    assert st["d2h_bytes"] == M * Nc * 8 and st["kernel_launches"] >= 1
    sess.reset_stats()
    sess.fromDense(torch.from_numpy(A).cuda(), blk).toTorch(M, Nc, blk)
    st = sess.stats()
    assert st["h2d_bytes"] < 64 * 1024 and st["d2h_bytes"] == 0  # descriptor tables only


@pytest.mark.parametrize("algo", [0, 1])
def test_product_of_dense_ingests_matches_block_by_block(algo):
    """For C-order A and B, fromDense(A) x fromDense(B) is the product of the datasets built with transposed_storage=True."""
    M, K, Nc, blk = 700, 600, 500, 128
    rng = np.random.default_rng(algo + 11)
    A, B = rng.uniform(-1, 1, (M, K)), rng.uniform(-1, 1, (K, Nc))

    def blocks(X):
        return [mb.MatrixBlock(i, j, mb.DenseMatrix.from_numpy(X[i * blk:(i + 1) * blk, j * blk:(j + 1) * blk], transposed_storage=True))
                for i in range(-(-X.shape[0] // blk)) for j in range(-(-X.shape[1] // blk))]

    with mb.MatfastSession(device=0, gemm_algo=algo) as s:
        dA, dB = s.fromDense(A, blk), s.fromDense(B, blk)
        assert _dump(dA) == _dump(s.createDataset(blocks(A)))
        got = _dump(dA.matrixMultiply(M, K, dB, K, Nc, blk))
        want = _dump(s.createDataset(blocks(A)).matrixMultiply(M, K, s.createDataset(blocks(B)), K, Nc, blk))
    assert got == want


def _mixed_blocks(M, Nc, blk, seed):
    """Dense column-major and row-major blocks, CSC and CSR blocks, absent blocks, ragged edges, one block smaller than its cell."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(-(-M // blk)):
        for j in range(-(-Nc // blk)):
            r, c = min(blk, M - i * blk), min(blk, Nc - j * blk)
            kind = (i * 5 + j) % 6
            if kind == 5:
                continue  # absent
            a = rng.uniform(-1, 1, (r, c))
            if kind == 0:
                m = mb.DenseMatrix.from_numpy(a)
            elif kind == 1:
                m = mb.DenseMatrix.from_numpy(a, transposed_storage=True)
            elif kind in (2, 3):
                m = _sparse(np.where(rng.uniform(0, 1, (r, c)) < 0.2, a, 0.0), csr=kind == 3)
            else:  # smaller than its cell: the rest of the cell reads as zeros
                m = mb.DenseMatrix.from_numpy(a[:max(1, r - 3), :max(1, c - 2)], transposed_storage=bool(j % 2))
            out.append(mb.MatrixBlock(i, j, m))
    return out


@pytest.mark.parametrize("host", [False, True], ids=["device", "host"])
def test_assembly_of_arbitrary_datasets(sess, host):
    M, Nc, blk = 333, 290, 64
    rows = _mixed_blocks(M, Nc, blk, 3)
    kinds = {type(b.matrix).__name__ + str(b.matrix.isTransposed) for b in rows}
    assert kinds == {"DenseMatrixFalse", "DenseMatrixTrue", "SparseMatrixFalse", "SparseMatrixTrue"}
    ds = sess.createHostDataset(rows) if host else sess.createDataset(rows)
    _check_all_out(ds, _assemble(ds, M, Nc, blk), blk)


def test_assembly_of_a_streamed_product_in_several_panels(sess):
    """A host-resident product of a streamed multiply, assembled through panels under a small stream_budget_mb."""
    n, blk = 2048, 256
    rng = np.random.default_rng(9)
    A, B = rng.uniform(-1, 1, (n, n)), rng.uniform(-1, 1, (n, n))
    C_ = sess.fromDense(A, blk, host=True).matrixMultiply(n, n, sess.fromDense(B, blk, host=True), n, n, blk)
    assert C_.isHost
    want = _assemble(C_, n, n, blk)
    try:
        sess.set_option("stream_budget_mb", 40)  # a block-row panel is 4 MiB of output and 4 MiB of staging
        sess.reset_stats()
        _check_all_out(C_, want, blk)
        assert sess.stats()["kernel_launches"] == 2 * 8 + 2  # toNumpy x 2: 8 one-block-row panels each; toTorch: 2 panels
    finally:
        sess.set_option("stream_budget_mb", 0)


def test_side_stream_producer_is_waited_for(sess):
    M, Nc, blk = 2048, 2048, 256
    x = torch.randn(M, Nc, dtype=torch.float64, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        t = x
        for _ in range(8):  # keeps the side stream busy well past the call
            t = t @ x * (1.0 / Nc)
        ds = sess.fromDense(t, blk)
    side.synchronize()
    assert np.array_equal(ds.toNumpy(M, Nc, blk), t.cpu().numpy())


def test_to_torch_is_ordered_before_the_next_torch_op(sess):
    M, Nc, blk = 1500, 1300, 256
    A = np.random.default_rng(12).uniform(-1, 1, (M, Nc))
    ds = sess.fromDense(A, blk)
    got = (ds.toTorch(M, Nc, blk) * 2.0).cpu().numpy()  # no host sync between the assembly and the multiply
    assert np.array_equal(got, 2.0 * A)


def test_multiply_right_after_pinned_ingest(sess):
    n, blk = 2048, 256
    rng = np.random.default_rng(13)
    A, B = rng.uniform(-1, 1, (n, n)), rng.uniform(-1, 1, (n, n))
    want = _dump(sess.fromDense(A, blk).matrixMultiply(n, n, sess.fromDense(B, blk), n, n, blk))
    pA, pB = torch.from_numpy(A).pin_memory(), torch.from_numpy(B).pin_memory()
    dA, dB = sess.fromDense(pA, blk), sess.fromDense(pB, blk)
    assert _dump(dA.matrixMultiply(n, n, dB, n, n, blk)) == want


def test_pinned_source_may_be_reused_after_wait_ingest(sess):
    M, Nc, blk = 1024, 768, 128
    A = np.random.default_rng(14).uniform(-1, 1, (M, Nc))
    p = torch.from_numpy(A.copy()).pin_memory()
    ds = sess.fromDense(p, blk)
    ds.wait_ingest()
    p.fill_(7.0)
    assert np.array_equal(ds.toNumpy(M, Nc, blk), A)


def test_errors_leave_the_session_usable(sess):
    A = np.random.default_rng(15).uniform(-1, 1, (100, 64))
    out = C.c_void_p()
    # ld below the contiguous dimension, through the C ABI (the façades derive ld from the strides)
    st = N.lib.mr_matrix_from_dense(sess._ctx, C.c_void_p(A.ctypes.data), 100, 64, 63, 1, 32, 0, None, C.byref(out))
    assert st == N.MR_EINVAL and "ld = 63 is smaller than the contiguous dimension 64" in N.last_error()
    ds = sess.fromDense(A, 32)
    st = N.lib.mr_matrix_to_dense(ds._h, 100, 64, 32, C.c_void_p(A.ctypes.data), 99, 0, None)
    assert st == N.MR_EINVAL and "ld = 99 is smaller than the contiguous dimension 100" in N.last_error()
    with pytest.raises(mb.IllegalArgumentException, match="nrows, ncols, blkSize must be positive"):
        sess.fromDense(A, 0)
    with pytest.raises(mb.IllegalArgumentException, match="nrows, ncols, blkSize must be positive"):
        ds.toNumpy(100, 64, -1)
    # a block outside the matrix
    with pytest.raises(mb.IllegalArgumentException, match=r"block \(3, 0\) of 4 x 32 does not lie inside the 99 x 64 matrix in blocks of 32"):
        ds.toNumpy(99, 64, 32)
    big = sess.createDataset([mb.MatrixBlock(0, 0, mb.DenseMatrix.from_numpy(np.ones((40, 8))))])
    with pytest.raises(mb.IllegalArgumentException, match=r"block \(0, 0\) of 40 x 8 does not lie inside the 100 x 64 matrix in blocks of 32"):
        big.toNumpy(100, 64, 32)
    # dtype, strides, devices
    with pytest.raises(TypeError, match="float64"):
        sess.fromDense(A.astype(np.float32), 32)
    with pytest.raises(TypeError, match="float64"):
        sess.fromDense(torch.zeros(4, 4, dtype=torch.float32, device="cuda"), 32)
    with pytest.raises(ValueError, match="one unit-stride dimension"):
        sess.fromDense(A[::2, ::2], 32)
    with pytest.raises(ValueError, match="CPU and CUDA tensors only"):
        sess.fromDense(torch.zeros(4, 4, dtype=torch.float64, device="meta"), 32)
    if torch.cuda.device_count() > 1:
        with pytest.raises(ValueError, match="the session runs on cuda:0"):
            sess.fromDense(torch.zeros(4, 4, dtype=torch.float64, device="cuda:1"), 32)
    # a host dst whose panel does not fit the budget
    h = sess.fromDense(A, 32, host=True)
    try:
        sess.set_option("stream_budget_mb", 1)
        big_h = sess.fromDense(np.zeros((4096, 4096)), 1024, host=True)
        with pytest.raises(MemoryError, match="one block-row panel needs .* bytes of device memory .* the budget is 1048576 bytes"):
            big_h.toNumpy(4096, 4096, 1024)
    finally:
        sess.set_option("stream_budget_mb", 0)
    # the session still works
    assert np.array_equal(h.toNumpy(100, 64, 32), A)
    assert np.array_equal(sess.fromDense(A, 32).toTorch(100, 64, 32).cpu().numpy(), A)
    sess.sync()

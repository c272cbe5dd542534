"""Device blocks whose base pointer is 8-byte but not 16-byte aligned: adopted through put_block_device at an odd element offset
of an allocation, or produced by vec() from a block with an odd number of rows.  The element-wise, reduction, fp64 GEMM and
Ozaki staging kernels have a separate path for such pointers (no 128-bit accesses); each is held to the tolerance its aligned
twin has in test_gpu_parity.py."""
import numpy as np
import pytest

import matrel_b200 as mb
from oracle import matrel_oracle as O
from tests.util import assert_same_dataset, from_dataset, random_block_dataset

pytestmark = pytest.mark.gpu


def adopt_unaligned(session, ds):
    """The dense block dict `ds` as a dataset whose blocks sit back to back from element 1 of one device allocation.
    Returns (dataset, tensor that owns the memory)."""
    import torch
    total = sum(m.values.size for m in ds.values())
    buf = torch.empty(total + 1, dtype=torch.float64, device="cuda")
    assert buf.data_ptr() % 16 == 0
    out, off, misaligned = session.emptyDataset(), 1, 0
    for (i, j), m in sorted(ds.items()):
        buf[off:off + m.values.size] = torch.from_numpy(m.values)
        ptr = buf.data_ptr() + 8 * off
        misaligned += ptr % 16 == 8
        out.put_block_device(i, j, m.numRows, m.numCols, ptr, m.isTransposed)
        off += m.values.size
    torch.cuda.synchronize()
    assert misaligned >= 1 and (buf.data_ptr() + 8) % 16 == 8
    return out, buf


@pytest.fixture(params=[(200, 168, 64), (199, 131, 67)], ids=["even", "odd"])
def pair(request, session):
    n, m, blk = request.param
    rng = np.random.default_rng(n)
    A = random_block_dataset(rng, n, m, blk, density=0.9, p_transposed=0.5, lo=0.5, hi=2.0)
    B = random_block_dataset(rng, n, m, blk, density=0.9, p_transposed=0.5, lo=0.5, hi=2.0)
    dA, ka = adopt_unaligned(session, A)
    dB, kb = adopt_unaligned(session, B)
    yield n, m, blk, A, B, dA, dB
    del dA, dB, ka, kb


def check_elementwise(n, m, blk, A, B, dA, dB):
    assert_same_dataset(from_dataset(dA.addElement(n, m, dB, n, m, blk)), O.add_element(A, n, m, B, n, m, blk), tol=1e-15)
    assert_same_dataset(from_dataset(dA.multiplyElement(n, m, dB, n, m, blk)), O.multiply_element(A, n, m, B, n, m, blk), tol=1e-15)
    assert_same_dataset(from_dataset(dA.divideElement(n, m, dB, n, m, blk)), O.divide_element(A, n, m, B, n, m, blk), tol=1e-15)
    assert_same_dataset(from_dataset(dA.multiplyScalar(-2.25)), O.multiply_scalar(A, -2.25), exact_storage=True)
    assert_same_dataset(from_dataset(dA.power(2.0)), O.power(A, 2.0), tol=1e-15)
    assert_same_dataset(from_dataset(dA.power(-1.3)), O.power(A, -1.3), tol=1e-14)
    assert_same_dataset(from_dataset(dA.rowSum(n, m)), O.row_sum(A, n, m), tol=1e-14)
    assert_same_dataset(from_dataset(dA.colSum(n, m)), O.col_sum(A, n, m), tol=1e-14)
    assert_same_dataset(from_dataset(dA.sum(n, m)), O.total_sum(A, n, m), tol=1e-13)


def test_elementwise_and_reductions_on_unaligned_blocks(pair):
    check_elementwise(*pair)


def test_materialize_of_transposed_unaligned_blocks(pair):
    n, m, blk, A, _, dA, _ = pair
    mat = from_dataset(dA.t().materialize())
    for key, want in O.transpose(A).items():
        g = mat[key]
        assert isinstance(g, mb.DenseMatrix) and not g.isTransposed
        assert np.array_equal(g.to_numpy(), want.to_numpy())


@pytest.mark.parametrize("algo,tol", [(1, 1e-11), (4, 1e-13)])
def test_multiply_of_unaligned_blocks(session, algo, tol):
    for (n, k, m, blk) in ((200, 168, 136, 64), (199, 131, 93, 67)):
        rng = np.random.default_rng(n + algo)
        A = random_block_dataset(rng, n, k, blk, p_transposed=0.5)
        B = random_block_dataset(rng, k, m, blk, p_transposed=0.5)
        with mb.MatfastSession(device=0, gemm_algo=algo) as s:
            dA, ka = adopt_unaligned(s, A)
            dB, kb = adopt_unaligned(s, B)
            got = from_dataset(dA.matrixMultiply(n, k, dB, k, m, blk))
            assert s.stats()["tc_gemm_launches"] == (1 if algo == 4 else 0)
            del dA, dB
        assert_same_dataset(got, O.matrix_multiply(A, n, k, B, k, m, blk), tol=tol)


def test_elementwise_on_vec_of_a_block_with_odd_rows(session):
    """vec() of a 67 x c block yields c column blocks of 67 rows carved out of one allocation: every other one starts at an odd
    element offset."""
    rng = np.random.default_rng(6)
    n, m, blk = 67, 40, 67
    A = random_block_dataset(rng, n, m, blk, lo=0.5, hi=2.0)
    B = random_block_dataset(rng, n, m, blk, lo=0.5, hi=2.0)
    vA, vB = O.vec(A, n, m, blk), O.vec(B, n, m, blk)
    dA = session.createDataset(mb.MatrixBlock(i, j, mb.DenseMatrix(x.numRows, x.numCols, x.values, x.isTransposed)) for (i, j), x in A.items()).vec(n, m, blk)
    dB = session.createDataset(mb.MatrixBlock(i, j, mb.DenseMatrix(x.numRows, x.numCols, x.values, x.isTransposed)) for (i, j), x in B.items()).vec(n, m, blk)
    assert any(dA.block_device_ptr(*key) % 16 == 8 for key in dA.block_ids())
    check_elementwise(n * m, 1, blk, vA, vB, dA, dB)

"""GPU tests of the fp32 multiply on wgmma tf32 (gemm_algo = 3, 3xTF32 split) -- BASELINE configs[3] shape.

fp32 is not a reference feature (blocks are Array[Double]); parity is defined as: inputs rounded to fp32, oracle =
fp64 product of those inputs, tolerance 1e-5 relative to max|C| (the north-star bar).  What makes it hold: the 3xTF32 split,
K chunks of 2048 re-accumulated in fp64, and -- for operands fully covered by blocks -- mean-centring: the tensor core's fp32
accumulation truncates, a bias that grows with K for same-signed data (1e-4 at K = 16384 on U(0,1) inputs); the operand means
are removed before the split and put back in fp64 by the epilogue.  (A single-pass TF32 product would be ~1e-3.)"""
import numpy as np
import pytest

import matrel_b200 as mb
from oracle import matrel_oracle as O
from tests.util import assert_same_dataset, from_dataset, random_block_dataset, rel_err, to_dataset

pytestmark = pytest.mark.gpu
TF32X3_TOL = 1e-5


def f32_round(ds):
    out = {}
    for k, m in ds.items():
        out[k] = O.DenseMatrix(m.numRows, m.numCols, m.values.astype(np.float32).astype(np.float64), m.isTransposed)
    return out


def test_tf32x3_positive_data_long_k():
    """All-positive U(0,1) data at K = 16384: the worst case for fp32 accumulation drift."""
    n, blk = 16384, 1024
    with mb.MatfastSession(device=0, gemm_algo=3) as s:
        A, B = s.rand(n, n, blk, 42), s.rand(n, n, blk, 43)
        C = A.matrixMultiply(n, n, B, n, n, blk)
        a = np.concatenate([A.get_block(0, k).to_numpy().astype(np.float32).astype(np.float64) for k in range(n // blk)], axis=1)[:128]
        b = np.concatenate([B.get_block(k, 0).to_numpy().astype(np.float32).astype(np.float64) for k in range(n // blk)], axis=0)[:, :128]
        got = C.get_block(0, 0).to_numpy()[:128, :128]
    assert rel_err(got, a @ b) <= TF32X3_TOL


@pytest.mark.parametrize("n,k,m,blk,pt", [(256, 256, 256, 128, 0.0), (512, 640, 384, 128, 0.5), (300, 200, 260, 128, 0.5),
                                          (2048, 2048, 2048, 512, 0.3), (256, 9000, 256, 1000, 0.3)])
def test_tf32x3_multiply(n, k, m, blk, pt):
    rng = np.random.default_rng(n + k + m)
    A = f32_round(random_block_dataset(rng, n, k, blk, p_transposed=pt))
    B = f32_round(random_block_dataset(rng, k, m, blk, p_transposed=pt))
    want = O.matrix_multiply(A, n, k, B, k, m, blk)
    with mb.MatfastSession(device=0, gemm_algo=3) as s:
        got = from_dataset(to_dataset(s, A).matrixMultiply(n, k, to_dataset(s, B), k, m, blk))
        # one stats pass over both operands and its reduction, two slicing passes, the correction kernel (the operands are fully
        # covered, so centred), one wgmma launch per K chunk
        assert s.stats()["kernel_launches"] == 5 + -(-k // 2048)
    assert_same_dataset(got, want, tol=TF32X3_TOL)          # ids / presence / shapes / flags exact
    full_g = O.assemble({k_: O.DenseMatrix(v.numRows, v.numCols, v.values) for k_, v in got.items()}, n, m, blk)
    err = rel_err(full_g, O.assemble(want, n, m, blk))
    assert err <= TF32X3_TOL, err
    assert err > 0                                           # it really is fp32 arithmetic

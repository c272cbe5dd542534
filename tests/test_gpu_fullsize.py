"""Parity at the metric sizes through a size-independent property that touches EVERY block of the result (Freivalds' check):
for a random vector x,  C x  must equal  A (B x)  -- both sides computed by the engine itself from the device-resident blocks
with O(N^2) work, compared on the host over all N rows.  A wrong, missing or misplaced output block, or a wrong k-reduction,
changes C x by O(|C|); the tolerance is 1e-11 of the row's magnitude (the north-star bar is 1e-5).  The exact kernel that
multiplies by x is the fp64 DMMA kernel (small products stay on it), so the check is independent of the wgmma path."""
import numpy as np
import pytest

import matrel_b200 as mb

pytestmark = pytest.mark.gpu


def _vector_dataset(session, x, blk):
    n = x.size
    return session.createDataset(mb.MatrixBlock(i, 0, mb.DenseMatrix(min(blk, n - i * blk), 1, x[i * blk:(i + 1) * blk].copy()))
                                 for i in range(-(-n // blk)))


def _collect_vector(ds, n, blk):
    out = np.zeros(n)
    for b in ds.collect():
        assert b.cid == 0 and b.matrix.numCols == 1
        out[b.rid * blk:b.rid * blk + b.matrix.numRows] = b.matrix.to_numpy()[:, 0]
    return out


@pytest.mark.parametrize("n,blk,algo", [(16384, 1024, 1), (16384, 1024, 0), (32768, 2048, 0)])
def test_freivalds_every_block(n, blk, algo):
    import torch
    free, _ = torch.cuda.mem_get_info(0)
    need = 3 * n * n * 8 + (18 << 30)
    if free < need:
        pytest.skip(f"needs {need >> 30} GiB of device memory")
    rng = np.random.default_rng(n + algo)
    with mb.MatfastSession(device=0, gemm_algo=algo) as s:
        A, B = s.rand(n, n, blk, 42), s.rand(n, n, blk, 43)
        s.reset_stats()
        C = A.matrixMultiply(n, n, B, n, n, blk)
        st = s.stats()
        assert (st["tc_gemm_launches"] == 1) == (algo == 0)          # auto: the wgmma path; 1: the DMMA kernel
        assert len(C.block_ids()) == (n // blk) ** 2
        s.set_option("gemm_algo", 1)                                   # the checker's mat-vecs: exact kernel
        for trial in range(2):
            x = rng.uniform(-1, 1, n)
            dx = _vector_dataset(s, x, blk)
            Bx = B.matrixMultiply(n, n, dx, n, 1, blk)
            ABx = _collect_vector(A.matrixMultiply(n, n, Bx, n, 1, blk), n, blk)
            Cx = _collect_vector(C.matrixMultiply(n, n, dx, n, 1, blk), n, blk)
            scale = np.abs(ABx) + n * 1e-3                             # entries of A (B x) are sums of n terms of size ~0.25 n
            assert np.max(np.abs(Cx - ABx) / scale) <= 1e-11, (trial, float(np.max(np.abs(Cx - ABx) / scale)))
        # and the row sums through the aggregate operator: (A B) 1 = A (B 1)
        ones = _vector_dataset(s, np.ones(n), blk)
        AB1 = _collect_vector(A.matrixMultiply(n, n, B.matrixMultiply(n, n, ones, n, 1, blk), n, 1, blk), n, blk)
        rs = _collect_vector(C.rowSum(n, n), n, blk)
        assert np.max(np.abs(rs - AB1) / np.abs(AB1)) <= 1e-11

"""GPU tests of the wgmma (s8) Ozaki fp64 multiply (gemm_algo = 2) against the CPU oracle.

The path is an fp64 emulation: every slice product is an exact integer GEMM; the error comes from the
final digit of the per-row / per-column aligned slicing.  Bars: north_star's 1e-5 relative, and a much
tighter per-slice-count bound (relative to max|C|) so that a broken slice/diagonal cannot hide."""
import numpy as np
import pytest

import matrel_b200 as mb
from oracle import matrel_oracle as O
from tests.util import REL_TOL, assert_same_dataset, from_dataset, random_block_dataset, rel_err, to_dataset

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def oz():
    s = mb.MatfastSession(device=0, gemm_algo=2, ozaki_slices=7)
    yield s
    s.stop()


def full(ds, n, m, blk):
    out = np.zeros((n, m))
    for (i, j), b in ds.items():
        out[i * blk:i * blk + b.numRows, j * blk:j * blk + b.numCols] = b.to_numpy()
    return out


@pytest.mark.parametrize("n,k,m,blk,pt", [
    (256, 256, 256, 128, 0.0),
    (512, 384, 640, 128, 0.5),      # all four T/N combinations, several 128x256 tiles
    (300, 200, 260, 128, 0.5),      # ragged edges
    (131, 77, 93, 64, 0.5),         # odd dims: byte-wise slice stores at block edges
    (1024, 1024, 1024, 256, 0.3),   # BASELINE config[0] shape
])
def test_ozaki_multiply_vs_oracle(oz, n, k, m, blk, pt):
    rng = np.random.default_rng(n + 3 * k + 7 * m + blk)
    A = random_block_dataset(rng, n, k, blk, p_transposed=pt)
    B = random_block_dataset(rng, k, m, blk, p_transposed=pt)
    want = O.matrix_multiply(A, n, k, B, k, m, blk)
    oz.reset_stats()
    got = from_dataset(to_dataset(oz, A).matrixMultiply(n, k, to_dataset(oz, B), k, m, blk))
    assert oz.stats()["kernel_launches"] >= 5 + 7          # absmax x2, exp, slice x2, one GEMM per diagonal
    assert_same_dataset(got, want, tol=REL_TOL)            # ids / presence / shapes / flags exact
    err = rel_err(full(got, n, m, blk), full(want, n, m, blk))
    assert err <= 1e-13, err                               # 7 slices: fp64-rounding level for U(-1,1) data


@pytest.mark.parametrize("slices,bound", [(3, 2e-5), (4, 1e-7), (5, 5e-10), (6, 2e-12), (7, 1e-13)])
def test_ozaki_error_scales_with_slices(slices, bound):
    rng = np.random.default_rng(slices)
    n, blk = 512, 128
    A = random_block_dataset(rng, n, n, blk, lo=0.0, hi=1.0)
    B = random_block_dataset(rng, n, n, blk, lo=0.0, hi=1.0)
    want = full(O.matrix_multiply(A, n, n, B, n, n, blk), n, n, blk)
    with mb.MatfastSession(device=0, gemm_algo=2, ozaki_slices=slices) as s:
        got = full(from_dataset(to_dataset(s, A).matrixMultiply(n, n, to_dataset(s, B), n, n, blk)), n, n, blk)
    assert rel_err(got, want) <= bound, rel_err(got, want)


def test_ozaki_wide_dynamic_range_rows_and_columns(oz):
    """Rows of A and columns of B scaled over 2^-40 .. 2^40: the per-row / per-column exponents absorb it."""
    rng = np.random.default_rng(17)
    n, blk = 384, 128
    Af = rng.uniform(-1, 1, (n, n)) * np.exp2(rng.integers(-40, 40, n))[:, None]
    Bf = rng.uniform(-1, 1, (n, n)) * np.exp2(rng.integers(-40, 40, n))[None, :]

    def blocks(M):
        return {(i, j): O.DenseMatrix(blk, blk, np.ascontiguousarray(M[i * blk:(i + 1) * blk, j * blk:(j + 1) * blk].T).reshape(-1))
                for i in range(n // blk) for j in range(n // blk)}
    got = full(from_dataset(to_dataset(oz, blocks(Af)).matrixMultiply(n, n, to_dataset(oz, blocks(Bf)), n, n, blk)), n, n, blk)
    want = Af @ Bf
    scale = np.abs(Af) @ np.abs(Bf)
    assert np.max(np.abs(got - want) / scale) <= 1e-12


def test_ozaki_block_sparse_presence_and_zero_rows(oz):
    rng = np.random.default_rng(23)
    n, blk = 5 * 64, 64
    A = random_block_dataset(rng, n, n, blk, density=0.5, p_transposed=0.3)
    B = random_block_dataset(rng, n, n, blk, density=0.5, p_transposed=0.3)
    key = next(iter(A))
    A[key] = O.DenseMatrix(A[key].numRows, A[key].numCols, np.zeros(A[key].numRows * A[key].numCols))  # all-zero block
    want = O.matrix_multiply(A, n, n, B, n, n, blk)
    got = from_dataset(to_dataset(oz, A).matrixMultiply(n, n, to_dataset(oz, B), n, n, blk))
    assert_same_dataset(got, want, tol=1e-12)


def test_ozaki_nonfinite_falls_back_to_exact_kernel(oz):
    n, blk = 256, 128
    A = O.rand_dense_dataset(n, n, blk, 1)
    B = O.rand_dense_dataset(n, n, blk, 2)
    A[(0, 0)].values[5] = np.inf
    want = O.matrix_multiply(A, n, n, B, n, n, blk)
    got = from_dataset(to_dataset(oz, A).matrixMultiply(n, n, to_dataset(oz, B), n, n, blk))
    assert_same_dataset(got, want, tol=1e-12)


def test_ozaki_matches_dmma_at_4096(oz, session):
    n, blk = 4096, 512
    A1, B1 = session.rand(n, n, blk, 42), session.rand(n, n, blk, 43)
    A2, B2 = oz.rand(n, n, blk, 42), oz.rand(n, n, blk, 43)
    C1 = A1.matrixMultiply(n, n, B1, n, n, blk)
    C2 = A2.matrixMultiply(n, n, B2, n, n, blk)
    worst = 0.0
    for key in C1.block_ids():
        a, b = C1.get_block(*key).values, C2.get_block(*key).values
        worst = max(worst, float(np.max(np.abs(a - b)) / np.max(np.abs(a))))
    assert worst <= 1e-13, worst

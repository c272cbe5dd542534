"""GPU tests of the Ozaki scheme II fp64 multiply (gemm_algo = 4: int8 wgmma GEMMs of residue matrices + CRT).

The integer product of the scaled operands is recovered EXACTLY, so (a) integer-valued inputs give bit-exact
results, and (b) the only error is the rounding of the operands to alpha bits relative to their row / column
maximum plus one final rounding.  The number of moduli follows the inner dimension (crt_moduli = 0, the default:
14 moduli, alpha = 54 - ceil(lg K / 2) or better, so sqrt(K) 2^-alpha stays below half the fp64 dot-product bound
K 2^-53); 16 moduli (alpha >= 53 for K <= 2^16) can be requested.  Bars: bit-exact for integer data; 1e-14
relative to |A||B| at the default and at 16 moduli."""
import numpy as np
import pytest

import matrel_b200 as mb
from oracle import matrel_oracle as O
from tests.util import REL_TOL, assert_same_dataset, from_dataset, random_block_dataset, rel_err, to_dataset

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def oz2():
    s = mb.MatfastSession(device=0, gemm_algo=4)
    yield s
    s.stop()


def full(ds, n, m, blk):
    out = np.zeros((n, m))
    for (i, j), b in ds.items():
        out[i * blk:i * blk + b.numRows, j * blk:j * blk + b.numCols] = b.to_numpy()
    return out


def blocks_of(M, blk):
    n, m = M.shape
    out = {}
    for i in range((n + blk - 1) // blk):
        for j in range((m + blk - 1) // blk):
            sub = M[i * blk:(i + 1) * blk, j * blk:(j + 1) * blk]
            out[(i, j)] = O.DenseMatrix(sub.shape[0], sub.shape[1], np.ascontiguousarray(sub.T).reshape(-1))
    return out


@pytest.mark.parametrize("n,k,m,blk,pt", [
    (256, 256, 256, 128, 0.0),
    (512, 384, 640, 128, 0.5),      # all four T/N combinations, several 128x256 tiles
    (300, 200, 260, 128, 0.5),      # ragged edges
    (131, 77, 93, 64, 0.5),         # odd dims: byte-wise residue stores at block edges
    (1024, 1024, 1024, 256, 0.3),   # BASELINE config[0] shape
])
def test_crt_multiply_vs_oracle(oz2, n, k, m, blk, pt):
    rng = np.random.default_rng(n + 3 * k + 7 * m + blk)
    A = random_block_dataset(rng, n, k, blk, p_transposed=pt)
    B = random_block_dataset(rng, k, m, blk, p_transposed=pt)
    want = O.matrix_multiply(A, n, k, B, k, m, blk)
    oz2.reset_stats()
    got = from_dataset(to_dataset(oz2, A).matrixMultiply(n, k, to_dataset(oz2, B), k, m, blk))
    assert oz2.stats()["kernel_launches"] >= 7             # absmax x2, exp, residues x2, ONE GEMM launch, CRT
    assert_same_dataset(got, want, tol=REL_TOL)            # ids / presence / shapes / flags exact
    err = rel_err(full(got, n, m, blk), full(want, n, m, blk))
    assert err <= 1e-14, err


@pytest.mark.parametrize("n,k,m,blk", [(256, 384, 256, 128), (200, 333, 150, 64)])
def test_crt_is_bit_exact_on_integer_data(oz2, n, k, m, blk):
    """Integers below 2^20: every product and sum is exact in fp64 AND in the residue arithmetic -> identical bits."""
    rng = np.random.default_rng(5)
    Af = rng.integers(-(1 << 20), 1 << 20, (n, k)).astype(np.float64)
    Bf = rng.integers(-(1 << 20), 1 << 20, (k, m)).astype(np.float64)
    got = full(from_dataset(to_dataset(oz2, blocks_of(Af, blk)).matrixMultiply(n, k, to_dataset(oz2, blocks_of(Bf, blk)), k, m, blk)), n, m, blk)
    want = (Af.astype(object) @ Bf.astype(object)).astype(np.float64)   # exact integer product (|c| < 2^50)
    assert np.array_equal(got, want)


@pytest.mark.parametrize("moduli,bound", [(8, 2e-7), (10, 1e-9), (12, 5e-12), (14, 2e-14), (16, 5e-15)])
def test_crt_error_scales_with_moduli(moduli, bound):
    rng = np.random.default_rng(moduli)
    n, blk = 512, 128
    A = random_block_dataset(rng, n, n, blk, lo=0.0, hi=1.0)
    B = random_block_dataset(rng, n, n, blk, lo=0.0, hi=1.0)
    want = full(O.matrix_multiply(A, n, n, B, n, n, blk), n, n, blk)
    with mb.MatfastSession(device=0, gemm_algo=4) as s:
        s.set_option("crt_moduli", moduli)
        got = full(from_dataset(to_dataset(s, A).matrixMultiply(n, n, to_dataset(s, B), n, n, blk)), n, n, blk)
    assert rel_err(got, want) <= bound, rel_err(got, want)


def test_default_moduli_follow_the_inner_dimension(oz2):
    rng = np.random.default_rng(41)
    n, blk = 1024, 256
    Af, Bf = rng.uniform(-1, 1, (n, n)), rng.uniform(-1, 1, (n, n))
    want, scale = Af @ Bf, np.abs(Af) @ np.abs(Bf)
    errs = {}
    for moduli in (0, 16):
        with mb.MatfastSession(device=0, gemm_algo=4) as s:
            s.set_option("crt_moduli", moduli)
            got = full(from_dataset(to_dataset(s, blocks_of(Af, blk)).matrixMultiply(n, n, to_dataset(s, blocks_of(Bf, blk)), n, n, blk)), n, n, blk)
            assert s.stats()["tc_moduli"] == (moduli or 14)
            errs[moduli] = float(np.max(np.abs(got - want) / scale))
    # both sit at the rounding level of the fp64 reference product itself (|A||B|-relative)
    assert errs[16] <= 5e-16 and errs[0] <= 1e-15, errs


def test_crt_wide_dynamic_range_rows_and_columns(oz2):
    rng = np.random.default_rng(17)
    n, blk = 384, 128
    Af = rng.uniform(-1, 1, (n, n)) * np.exp2(rng.integers(-40, 40, n))[:, None]
    Bf = rng.uniform(-1, 1, (n, n)) * np.exp2(rng.integers(-40, 40, n))[None, :]
    got = full(from_dataset(to_dataset(oz2, blocks_of(Af, blk)).matrixMultiply(n, n, to_dataset(oz2, blocks_of(Bf, blk)), n, n, blk)), n, n, blk)
    want = Af @ Bf
    scale = np.abs(Af) @ np.abs(Bf)
    assert np.max(np.abs(got - want) / scale) <= 1e-14


def test_crt_block_sparse_presence_and_zero_rows(oz2):
    rng = np.random.default_rng(23)
    n, blk = 5 * 64, 64
    A = random_block_dataset(rng, n, n, blk, density=0.5, p_transposed=0.3)
    B = random_block_dataset(rng, n, n, blk, density=0.5, p_transposed=0.3)
    key = next(iter(A))
    A[key] = O.DenseMatrix(A[key].numRows, A[key].numCols, np.zeros(A[key].numRows * A[key].numCols))  # all-zero block
    want = O.matrix_multiply(A, n, n, B, n, n, blk)
    got = from_dataset(to_dataset(oz2, A).matrixMultiply(n, n, to_dataset(oz2, B), n, n, blk))
    assert_same_dataset(got, want, tol=1e-13)


def test_crt_nonfinite_falls_back_to_exact_kernel(oz2):
    n, blk = 256, 128
    A = O.rand_dense_dataset(n, n, blk, 1)
    B = O.rand_dense_dataset(n, n, blk, 2)
    A[(0, 0)].values[5] = np.nan
    want = O.matrix_multiply(A, n, n, B, n, n, blk)
    got = from_dataset(to_dataset(oz2, A).matrixMultiply(n, n, to_dataset(oz2, B), n, n, blk))
    assert_same_dataset(got, want, tol=1e-12)


def test_crt_matches_dmma_at_4096(oz2, session):
    n, blk = 4096, 512
    A1, B1 = session.rand(n, n, blk, 42), session.rand(n, n, blk, 43)
    A2, B2 = oz2.rand(n, n, blk, 42), oz2.rand(n, n, blk, 43)
    C1 = A1.matrixMultiply(n, n, B1, n, n, blk)
    C2 = A2.matrixMultiply(n, n, B2, n, n, blk)
    worst = 0.0
    for key in C1.block_ids():
        a, b = C1.get_block(*key).values, C2.get_block(*key).values
        worst = max(worst, float(np.max(np.abs(a - b)) / np.max(np.abs(a))))
    assert worst <= 2e-14, worst      # the deviation is the DMMA kernel's own accumulated rounding (K = 4096)


# ---------------------------------------------------------------------------------- job engine
def _pinned_blocks(ds):
    import torch
    pin = lambda m: mb.DenseMatrix(m.numRows, m.numCols, torch.from_numpy(m.values).pin_memory().numpy(), m.isTransposed)  # noqa: E731
    return [mb.MatrixBlock(i, j, pin(m)) for (i, j), m in ds.items()]


def test_crt_pipelined_behind_ingest_is_bit_identical(oz2):
    """The tensor-core path runs chunk by chunk behind the host->device ingest (residues of a block row / column as soon as it is
    complete, int8 GEMM + CRT of the output blocks it unlocks).  Row / column exponents do not depend on the chunking and the
    integer product is exact, so the blocks must equal the resident run's bit for bit -- whatever order the blocks arrive in."""
    n, blk = 2048, 256
    nb = n // blk
    A = O.rand_dense_dataset(n, n, blk, 42, transposed_mask=lambda i, j: (i * 3 + j) % 4 == 0)
    B = O.rand_dense_dataset(n, n, blk, 43)
    ref = from_dataset(to_dataset(oz2, A).matrixMultiply(n, n, to_dataset(oz2, B), n, n, blk))
    want = O.matrix_multiply(A, n, n, B, n, n, blk)
    assert_same_dataset(ref, want, tol=1e-13)
    pA, pB = _pinned_blocks(A), _pinned_blocks(B)
    rowsA = {t: [b for b in pA if b.rid == t] for t in range(nb)}
    colsB = {t: [b for b in pB if b.cid == t] for t in range(nb)}
    for order in ("alternate", "b_first", "a_first"):
        oz2.reset_stats()
        dA, dB = oz2.emptyDataset(), oz2.emptyDataset()
        if order == "alternate":
            for t in range(nb):
                dA.put_blocks(rowsA[t])
                dB.put_blocks(colsB[t])
        elif order == "b_first":
            dB.put_blocks(pB)
            dA.put_blocks(pA)
        else:
            dA.put_blocks(pA)
            dB.put_blocks(pB)
        got = from_dataset(dA.matrixMultiply(n, n, dB, n, n, blk))
        assert oz2.stats()["tc_gemm_launches"] == 1, order
        assert_same_dataset(got, {k: O.DenseMatrix(v.numRows, v.numCols, v.values) for k, v in ref.items()}, exact_storage=True)


def test_crt_panelled_scratch_is_bit_identical():
    """Operands whose residues exceed the scratch budget are multiplied as (row panel x column panel) jobs that re-prepare their
    slots; same bits as the resident run.  (Budgets of 6 / 12 / 24 MiB at n ~ 1024, blk = 128 give 1 x 1 up to 4 x 4-slot panels; everything resident needs 40 MiB.)"""
    rng = np.random.default_rng(99)
    n, k, m, blk = 1024 - 40, 768, 1024 - 100, 128
    A = random_block_dataset(rng, n, k, blk, p_transposed=0.4)
    B = random_block_dataset(rng, k, m, blk, p_transposed=0.4)
    with mb.MatfastSession(device=0, gemm_algo=4) as s:
        ref = from_dataset(to_dataset(s, A).matrixMultiply(n, k, to_dataset(s, B), k, m, blk))
        for mbytes in (6, 12, 24):
            s.set_option("ozaki_scratch_mb", mbytes)
            s.reset_stats()
            got = from_dataset(to_dataset(s, A).matrixMultiply(n, k, to_dataset(s, B), k, m, blk))
            assert s.stats()["tc_gemm_launches"] == 1
            assert_same_dataset(got, {kk: O.DenseMatrix(v.numRows, v.numCols, v.values) for kk, v in ref.items()}, exact_storage=True)
    assert_same_dataset(ref, O.matrix_multiply(A, n, k, B, k, m, blk), tol=1e-13)


def _adversarial(rng, n, tiny):
    """Row i of A = (1, tiny, tiny, ...), column j of B = (0, 1, 1, ...): |A||B|_ij = (n - 1) * tiny, carried ONLY by elements
    2^-60 below their row maximum -- the per-row scaling of the residue scheme rounds them away."""
    Af = np.full((n, n), tiny) * rng.uniform(1.0, 2.0, (n, n))
    Af[:, 0] = 1.0
    Bf = rng.uniform(1.0, 2.0, (n, n))
    Bf[0, :] = 0.0
    return Af, Bf


def test_auto_selection_guards_in_row_dynamic_range():
    """gemm_algo 0 (auto): the tensor-core path is taken for data of ordinary range (element-wise error <= 1e-13 |A||B|) and
    refused ON THE DEVICE when a non-zero element lies too far below its row / column maximum -- the exact DMMA kernel then
    runs instead and the element-wise bound against |A||B| holds.  gemm_algo 4 (unguarded) shows why the guard exists."""
    rng = np.random.default_rng(7)
    n, blk = 2048, 256
    with mb.MatfastSession(device=0, gemm_algo=0) as s:
        # ordinary data: in-row range of U(-1,1) over 2048 elements is ~2^-12..2^-25
        Af, Bf = rng.uniform(-1, 1, (n, n)), rng.uniform(-1, 1, (n, n))
        s.reset_stats()
        got = full(from_dataset(to_dataset(s, blocks_of(Af, blk)).matrixMultiply(n, n, to_dataset(s, blocks_of(Bf, blk)), n, n, blk)), n, n, blk)
        assert s.stats()["tc_gemm_launches"] == 1            # large regular product: the tensor-core path was planned
        assert np.max(np.abs(got - Af @ Bf) / (np.abs(Af) @ np.abs(Bf))) <= 1e-13
        # adversarial rows: guard trips, DMMA result
        Af, Bf = _adversarial(rng, n, 2.0 ** -60)
        want, scale = Af @ Bf, np.abs(Af) @ np.abs(Bf)
        got = full(from_dataset(to_dataset(s, blocks_of(Af, blk)).matrixMultiply(n, n, to_dataset(s, blocks_of(Bf, blk)), n, n, blk)), n, n, blk)
        assert np.max(np.abs(got - want) / scale) <= 1e-12
        # a range the guard accepts (2^-30 below the maximum keeps 25+ bits): still within the north-star tolerance of |A||B|
        Af, Bf = _adversarial(rng, n, 2.0 ** -30)
        want, scale = Af @ Bf, np.abs(Af) @ np.abs(Bf)
        got = full(from_dataset(to_dataset(s, blocks_of(Af, blk)).matrixMultiply(n, n, to_dataset(s, blocks_of(Bf, blk)), n, n, blk)), n, n, blk)
        assert np.max(np.abs(got - want) / scale) <= 1e-5
    with mb.MatfastSession(device=0, gemm_algo=4) as s:          # unguarded: the tiny elements vanish
        Af, Bf = _adversarial(rng, n, 2.0 ** -60)
        want, scale = Af @ Bf, np.abs(Af) @ np.abs(Bf)
        got = full(from_dataset(to_dataset(s, blocks_of(Af, blk)).matrixMultiply(n, n, to_dataset(s, blocks_of(Bf, blk)), n, n, blk)), n, n, blk)
        assert np.max(np.abs(got - want) / scale) > 1e-2


def test_auto_selection_corrects_isolated_tiny_elements_exactly():
    """A handful of elements far below their row / column maximum (what any large random matrix contains by chance) do not send
    the multiply to the fallback: the residue pass leaves them out and their products are added exactly in fp64 afterwards.
    Here they are placed where they matter -- C(i0, j0) consists of nothing but such a product -- and every other element of
    the result must be bit-identical to the unguarded tensor-core run (proof that the tensor-core path was kept)."""
    rng = np.random.default_rng(19)
    n, blk = 2048, 256
    Af, Bf = rng.uniform(1.0, 2.0, (n, n)), rng.uniform(1.0, 2.0, (n, n))
    spots = [(5, 700, 33), (5, 1900, 33), (300, 12, 1500), (1999, 2047, 0), (1024, 1024, 1024)]   # (i0, k0, j0)
    for (i0, k0, j0) in spots:
        Af[i0, k0] = 2.0 ** -45 * rng.uniform(1.0, 2.0)             # tiny element of row i0 of A ...
    for j0 in {j for _, _, j in spots}:
        ks = [k for _, k, j in spots if j == j0]
        Bf[:, j0] = 0.0
        Bf[ks, j0] = rng.uniform(1.0, 2.0, len(ks))                  # ... facing the only non-zeros of column j0 of B
    Bf[77, 900] = 2.0 ** -50                                         # and a tiny element of B (column 900 is ordinary)
    Bf[700, 33] *= 2.0 ** -48                                        # a tiny b facing a tiny a: the pair must be counted once
    want, scale = Af @ Bf, np.abs(Af) @ np.abs(Bf)
    res = {}
    for algo in (0, 4):
        with mb.MatfastSession(device=0, gemm_algo=algo) as s:
            res[algo] = full(from_dataset(to_dataset(s, blocks_of(Af, blk)).matrixMultiply(n, n, to_dataset(s, blocks_of(Bf, blk)), n, n, blk)), n, n, blk)
            assert s.stats()["tc_gemm_launches"] == 1
    err0 = np.abs(res[0] - want) / scale
    err4 = np.abs(res[4] - want) / scale
    assert np.max(err0) <= 1e-13, np.max(err0)                      # exact where only the tiny products contribute
    assert np.max(err4) > 1e-3                                       # the unguarded run loses them
    touched = np.zeros((n, n), dtype=bool)
    for (i0, _, _) in spots:
        touched[i0, :] = True                                        # rows with a tiny a: C(i0, :) += a B(k0, :)
    touched[:, 900] = True                                           # column with the tiny b
    touched[:, 33] = True
    assert np.array_equal(res[0][~touched], res[4][~touched])


def test_auto_selection_small_products_stay_on_dmma(session):
    n, blk = 512, 128
    A, B = session.rand(n, n, blk, 1), session.rand(n, n, blk, 2)
    session.reset_stats()
    A.matrixMultiply(n, n, B, n, n, blk)
    st = session.stats()
    assert st["tc_gemm_launches"] == 0 and st["kernel_launches"] == 1

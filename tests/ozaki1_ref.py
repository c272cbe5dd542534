"""CPU model of the Ozaki-I fp64 multiply (gemm_algo 2, ozaki_gemm_f64 in csrc/gemm_ozaki.cu), and its element-wise error bound.

ozaki1_model() replays the device arithmetic step by step, so the kernel must equal it bit for bit:
  1. e_i = ilogb(max_k |a_ik|) + 1 per row of A, f_j likewise per column of B (0 for an all-zero line);
  2. X = rint_half_even(a 2^(8S-2-e)) split into S balanced base-256 digits, least significant first, carry folded into the next
     (slice_kernel); digit 1 is the most significant, a = 2^(e+2) sum_s A_s 2^-8s up to the rounding of X;
  3. acc_d = sum_{s+t=d} A_s B_t for d = 2 .. S+1, exact integers: every partial sum stays below S K 2^14 < 2^31, so numpy's
     fp64 matmuls of the digit matrices are exact in any order;
  4. t_d = acc_d 2^(e_i+f_j+4-8d) rounded once (np.ldexp is correctly rounded, like ldexp_int on the device), then C = t_{S+1} and
     C = C + t_d for d = S .. 2, one fp64 addition each.  Where e_i + f_j > SCALED_ABOVE the terms and sums are kept scaled by
     2^-(e_i+f_j) -- exact there, as no term comes near the sub-normals -- and the sum after d = 2 is multiplied by 2^(e_i+f_j)
     with one rounding, so that only a sum beyond the fp64 range overflows, not a top-digit term.
A zero accumulator gives +0, so an entry is -0 only when every one of its S terms is a negative number that rounds to -0.

ozaki1_bound() is independent of the model: it is the bound DESIGN section 4.1.1 states.

The operands are the dense arrays the kernel sees: a block of A counts (for its row's exponent too) only when some block of B
shares its k, and likewise for B -- seen_operands() builds them from the block dicts."""
import numpy as np

from oracle import matrel_oracle as O

SCALED_ABOVE = 1000   # OZ1_SCALED_ABOVE of csrc/gemm_ozaki.cu


def line_exponents(M, axis):
    """ilogb(max |line|) + 1 of every row (axis=1) or column (axis=0), 0 for all-zero lines."""
    return np.frexp(np.abs(M).max(axis=axis, initial=0.0))[1].astype(np.int64)


def digits(L, e, S):
    """L: lines x K (rows of A, or columns of B as rows), e: exponent per line -> int64 [S, lines, K], slice 0 most significant."""
    with np.errstate(under="ignore"):
        X = np.rint(np.ldexp(L, (8 * S - 2 - e)[:, None])).astype(np.int64)      # |X| <= 2^(8S-2): exact in int64
    out = np.empty((S,) + L.shape, dtype=np.int64)
    for s in range(S, 0, -1):
        dgt = ((X + 128) & 255) - 128
        X = (X - dgt) >> 8
        out[s - 1] = dgt
    assert not X.any()
    return out


def diagonals(DA, DB, S):
    """{d: sum_{s+t=d} A_s B_t} for d = 2 .. S+1 (DA: [S, n, K], DB: [S, m, K] digit arrays), exact, as fp64 arrays."""
    fa, fb = DA.astype(np.float64), DB.astype(np.float64)
    return {d: sum(fa[s - 1] @ fb[d - s - 1].T for s in range(max(1, d - S), min(S, d - 1) + 1)) for d in range(2, S + 2)}


def epilogue(acc, e, f, S, scaled_above=None):
    """C = t_{S+1}, then C += t_d for d = S .. 2, with t_d = acc_d 2^(e_i + f_j + 4 - 8d) rounded once; kept scaled by 2^-(e_i + f_j)
    where e_i + f_j > scaled_above (SCALED_ABOVE unless given; a value above 2048 turns the scaling off)."""
    ef = e[:, None] + f[None, :]
    k = np.where(ef > (SCALED_ABOVE if scaled_above is None else scaled_above), ef, 0)
    C = None
    with np.errstate(over="ignore", under="ignore"):
        for d in range(S + 1, 1, -1):
            t = np.ldexp(acc[d], ef + 4 - 8 * d - k)
            C = t if C is None else C + t
        return np.ldexp(C, k)


def clamp_slices(slices):
    """ozaki_slices as the library takes it: 0 (default) -> 7, else clamped to 2 .. 7."""
    return 7 if slices <= 0 else min(7, max(2, slices))


def ozaki1_model(A, B, S):
    """The device result of A (n x K) times B (K x m) with S slices, bit for bit."""
    A, B = np.asarray(A, dtype=np.float64), np.asarray(B, dtype=np.float64)
    S = clamp_slices(S)
    e, f = line_exponents(A, 1), line_exponents(B, 0)
    return epilogue(diagonals(digits(A, e, S), digits(B.T, f, S), S), e, f, S)


def ozaki1_bound(A, B, S, C=None):
    """Element-wise bound of |got - exact| for the Ozaki-I product of A (n x K) and B (K x m) with S slices.

    With u = 2^(2-8S), 2^(e_i-1) <= rowmax_i < 2^e_i and 2^(f_j-1) <= colmax_j < 2^f_j:
      operand rounding   u (rowmax_i sum_k |b_kj| + colmax_j sum_k |a_ik|) (1 + K u)   (|da_ik| <= 2^(e_i+1-8S) <= u rowmax_i)
      dropped diagonals  sum_{d=S+2..2S} (2S+1-d) K 2^14 2^(e_i+f_j+4-8d)              (2S+1-d digit pairs of |product| <= 2^14)
      fp64 additions     (S-2) 2^-53 sum_{d=3..S+1} (d-1) K 2^14 2^(e_i+f_j+4-8d)    (partial sums before t_2 is added)
                         + 2^-52 |C_ij|                                             (the last addition, the rest's own rounding)
      sub-normal terms   (S+1) 2^-1074                                             (t_d and sums below 2^-1022)
    with the first three parts taken (1 + 2^-52) times: the last addition also rounds their error.
    At S = 7 the dropped diagonals alone reach about 6 K 2^(e_i+f_j-54) <= 24 K 2^-54 rowmax_i colmax_j.
    C: the exact product or anything close to it; left out, |A||B| >= |C| is used.  Computed in long double, so that the bound
    itself does not overflow at the top of the fp64 range."""
    A, B = np.asarray(A, dtype=np.float64), np.asarray(B, dtype=np.float64)
    S = clamp_slices(S)
    K = A.shape[1]
    ld = np.longdouble
    with np.errstate(over="ignore", invalid="ignore"):
        absA, absB = np.abs(A), np.abs(B)
        rowmax, colmax = absA.max(axis=1, initial=0.0), absB.max(axis=0, initial=0.0)
        u = ld(2.0) ** (2 - 8 * S)
        op = rowmax.astype(ld)[:, None] * absB.astype(ld).sum(axis=0)[None, :] + absA.astype(ld).sum(axis=1)[:, None] * colmax.astype(ld)[None, :]
        op = op * u * (1 + K * u)
        e, f = line_exponents(A, 1), line_exponents(B, 0)
        E = np.ldexp(np.ones((len(e), len(f)), dtype=ld), e[:, None] + f[None, :])
        E[rowmax == 0.0, :] = 0
        E[:, colmax == 0.0] = 0
        p2 = lambda n: ld(2.0) ** n                                                          # noqa: E731
        drop = sum((2 * S + 1 - d) * p2(4 - 8 * d) for d in range(S + 2, 2 * S + 1)) * ld(K) * p2(14) * E
        adds = (S - 2) * p2(-53) * sum((d - 1) * p2(4 - 8 * d) for d in range(3, S + 2)) * ld(K) * p2(14) * E
        mag = np.abs(C) if C is not None else absA @ absB
        tot = (op + drop + adds) * (1 + p2(-52)) + p2(-52) * mag.astype(ld) + (S + 1) * p2(-1074)
        return np.minimum(tot, ld(np.finfo(np.float64).max)).astype(np.float64)


def seen_operands(A, B, n, k, m, blk):
    """The dense operands the Ozaki-I kernel multiplies: blocks that meet no block of the other operand are left out (zeros), so
    they set no line's exponent.  Under the outer product (one block column of A) every block meets every block."""
    outer = -(-k // blk) == 1
    krows, kcols = {kk for (kk, _) in B}, {kk for (_, kk) in A}
    used_a = {key: x for key, x in A.items() if outer or key[1] in krows}
    used_b = {key: x for key, x in B.items() if outer or key[0] in kcols}
    return O.assemble(used_a, n, k, blk), O.assemble(used_b, k, m, blk)

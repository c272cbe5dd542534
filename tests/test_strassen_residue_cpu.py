"""CPU checks of the arithmetic of the Ozaki-II Strassen route (matrel_b200/csrc/gemm_ozaki.cu: strassen_residue_kernel, str_byte and
crt_kernel<NCH, true>; DESIGN section 4.1.3).  Nothing here runs the product: the coefficient and term tables are read from the source
and replayed with Python integers, the fp32 steps of the residue fold emulated exactly."""
import os
import random
import re
from fractions import Fraction

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = open(os.path.join(ROOT, "matrel_b200", "csrc", "gemm_ozaki.cu")).read()
MODULI = [int(x) for x in re.search(r"kCrtModuli\[CRT_MAX_T\] = \{([^}]*)\}", SRC).group(1).split(",")]


def table(name, rows):
    body = re.search(name + r"\[%d\]\[4\] = \{(.*?)\};" % rows, SRC, re.S).group(1)
    vals = [int(v) for v in re.findall(r"-?\d+", body)]
    assert len(vals) == 4 * rows
    return [vals[4 * i:4 * i + 4] for i in range(rows)]


COEF_A, COEF_B = table("kStrassenA", 7), table("kStrassenB", 7)
TERMS = table("c_str_terms", 4)


def fold_byte(Y, p):
    """The residue fold of strassen_residue_kernel / residue_kernel for one exact integer Y, |Y| < 2^64: the int8 it stores."""
    U = abs(Y)
    assert U < 1 << 64
    x = sum(((U >> (8 * i)) & 255) * pow(256, i, p) for i in range(8))   # two dp4a
    assert x < 1 << 19
    ip = Fraction(float(np.float32(1.0) / np.float32(p)))
    q = round(Fraction(x) * ip)                 # fmaf(f, ip, 1.5 * 2^23) - 1.5 * 2^23: round half to even, exact below 2^22
    r = x - q * p                                # fmaf(-q, p, f): exact
    v = -r if Y < 0 else r
    b = v & 255                                  # low byte of r * sgn + 1.5 * 2^23
    return b - 256 if b >= 128 else b


def test_combination_residues_at_the_extremes():
    """Sums and differences of two scaled elements reach 2^(alpha + 1) <= 2^62 (the route needs alpha <= 61): the stored byte is
    congruent to the exact sum modulo every p and within [-128, 128] (p = 256: a tie +-128 is stored as -128, which is congruent)."""
    random.seed(5)
    for alpha in (47, 55, 61):
        top = 1 << alpha
        pairs = [(top, top), (-top, -top), (top, -top), (-top, top), (top, 0), (0, -top), (top, top - 1), (-top, 1 - top),
                 (top - 1, -(top - 1)), (128, 0), (-128, 0), (128, 128), (-384, 0), (top - 128, 128)]
        for _ in range(40):
            pairs.append((random.randint(-top, top), random.randint(-top, top)))
            x = random.randint(-top // 256, top // 256) * 256 + 128               # p = 256 ties
            pairs.append((x, random.choice([0, 256, -256])))
        for a, b in pairs:
            for Y in (a + b, a - b):
                assert abs(Y) <= 1 << 62
                for p in MODULI:
                    r = fold_byte(Y, p)
                    assert (r - Y) % p == 0, (alpha, a, b, p, r)
                    assert -128 <= r <= 127 and abs(r) <= p // 2, (Y, p, r)


def str_byte(a, b, c, d, p, four):
    """str_byte in uint32 arithmetic: (a + b + d - c) mod p, or (a + b) mod p, for bytes in [0, p)."""
    m = 0xFFFFFFFF
    s = a + b
    if four:
        s = (s + d + p - c) & m
        s = min(s, (s - 2 * p) & m)
    return min(s, (s - p) & m)


def test_crt_combine_mod_p():
    """Every two-term combination exhaustively and the four-term ones on a dense sample, including all extreme bytes."""
    rng = np.random.default_rng(7)
    for p in MODULI:
        for a in range(p):
            for b in (0, 1, p // 2, p - 2, p - 1):
                assert str_byte(a, b, 0, 0, p, False) == (a + b) % p
        ext = [0, 1, p // 2, p - 2, p - 1]
        for a in ext:
            for b in ext:
                for c in ext:
                    for d in ext:
                        assert str_byte(a, b, c, d, p, True) == (a + b + d - c) % p
        v = rng.integers(0, p, size=(4, 4000))
        for a, b, c, d in v.T.tolist():
            assert str_byte(a, b, c, d, p, True) == (a + b + d - c) % p


def test_term_tables_are_strassen():
    """The coefficient tables and the quadrant terms are Strassen's: C11 = M1 + M4 - M5 + M7, C12 = M3 + M5, C21 = M2 + M4,
    C22 = M1 - M2 + M3 + M6, with M1..M7 as 0..6 and the third term of a four-term quadrant subtracted."""
    assert TERMS == [[0, 3, 4, 6], [2, 4, 0, 0], [1, 3, 0, 0], [0, 2, 1, 5]]
    # quadrant q = 2 h + g of (line half, k half): A11 A12 A21 A22 and B11 B21 B12 B22
    A = ["A11", "A12", "A21", "A22"]
    B = ["B11", "B21", "B12", "B22"]
    want_a = [{"A11": 1, "A22": 1}, {"A21": 1, "A22": 1}, {"A11": 1}, {"A22": 1}, {"A11": 1, "A12": 1}, {"A21": 1, "A11": -1},
              {"A12": 1, "A22": -1}]
    want_b = [{"B11": 1, "B22": 1}, {"B11": 1}, {"B12": 1, "B22": -1}, {"B21": 1, "B11": -1}, {"B22": 1}, {"B11": 1, "B12": 1},
              {"B21": 1, "B22": 1}]
    for i in range(7):
        assert {A[q]: c for q, c in enumerate(COEF_A[i]) if c} == want_a[i]
        assert {B[q]: c for q, c in enumerate(COEF_B[i]) if c} == want_b[i]


def sym(x, p):
    r = x % p
    return r - p if r > p // 2 else r


def test_seven_products_give_the_residues_of_the_product():
    """For random integer matrices of the operand range: the seven products of the reduced quadrant combinations, combined per
    quadrant modulo p as the CRT kernel does, equal (A B) mod p for every modulus -- the exact route's residues, so the same bits."""
    random.seed(11)
    for trial in range(6):
        m2, k2, n2 = random.choice([(2, 3, 2), (3, 4, 5), (4, 2, 3)])
        alpha = random.choice([20, 47, 61])
        top = 1 << alpha
        A = [[random.choice([random.randint(-top, top), top, -top, 0]) for _ in range(2 * k2)] for _ in range(2 * m2)]
        B = [[random.choice([random.randint(-top, top), top, -top, 0]) for _ in range(2 * n2)] for _ in range(2 * k2)]
        C = [[sum(A[i][k] * B[k][j] for k in range(2 * k2)) for j in range(2 * n2)] for i in range(2 * m2)]
        # quadrant (h, g) of A: rows h m2 .., columns g k2 ..; of B (line = column): columns h n2 .., rows g k2 ..
        qa = lambda q, r, k: A[(q >> 1) * m2 + r][(q & 1) * k2 + k]   # noqa: E731
        qb = lambda q, c, k: B[(q & 1) * k2 + k][(q >> 1) * n2 + c]   # noqa: E731
        for p in MODULI:
            M = []
            for i in range(7):
                Ai = [[sym(sum(COEF_A[i][q] * qa(q, r, k) for q in range(4)), p) for k in range(k2)] for r in range(m2)]
                Bi = [[sym(sum(COEF_B[i][q] * qb(q, c, k) for q in range(4)), p) for k in range(k2)] for c in range(n2)]
                # the int8 GEMM: exact s32 products of residues, stored as [0, p)
                M.append([[sum(Ai[r][k] * Bi[c][k] for k in range(k2)) % p for c in range(n2)] for r in range(m2)])
            for quad in range(4):
                a, b, c, d = TERMS[quad]
                four = quad in (0, 3)
                for r in range(m2):
                    for col in range(n2):
                        got = str_byte(M[a][r][col], M[b][r][col], M[c][r][col] if four else 0, M[d][r][col] if four else 0, p, four)
                        want = C[(quad >> 1) * m2 + r][(quad & 1) * n2 + col] % p
                        assert got == want, (trial, p, quad, r, col)

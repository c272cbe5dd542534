"""CPU check of the integer residue reduction of the int8 GEMM epilogue (mod_s32 / add_mod_bytes / store_residues in
matrel_b200/csrc/gemm_ozaki.cu), restated operation by operation in numpy uint32 / uint64 arithmetic with the constants the
host fills in (mod_magic = floor(2^32 / p), mod_off = (-2^31) mod p), against Python's % for every modulus of kCrtModuli:
the plain form (v mod p) and the ADD form ((v mod p) + y) mod p of the K-split order's upper half, for y the byte stored for
the lower half."""
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = open(os.path.join(ROOT, "matrel_b200", "csrc", "gemm_ozaki.cu")).read()
MODULI = [int(x) for x in re.search(r"kCrtModuli\[CRT_MAX_T\] = \{([^}]*)\}", SRC).group(1).split(",")]
U32 = np.uint64(0xFFFFFFFF)


def host_constants(p):
    """oz2_multiply: p.mod_magic[t] = (1 << 32) / p, p.mod_off[t] = (p - (1 << 31) % p) % p (uint32 arithmetic)."""
    return (1 << 32) // p, (p - (1 << 31) % p) % p


def umin(a, b):
    return np.minimum(a, b)


def mod_s32(v, p, magic, off):
    """mod_s32, every intermediate a uint32 (held in uint64 and wrapped with & 0xFFFFFFFF where the device wraps)."""
    p, magic, off = np.uint64(p), np.uint64(magic), np.uint64(off)
    w = (v.astype(np.int64) & 0xFFFFFFFF).astype(np.uint64) ^ np.uint64(0x80000000)   # static_cast<uint32_t>(v) ^ 0x80000000u
    q = (w * magic) >> np.uint64(32)                                                      # __umulhi(w, magic)
    r = (w - q * p) & U32
    r = umin(r, (r - p) & U32)
    r = (r + off) & U32
    return umin(r, (r - p) & U32)


def add_mod_byte(x, y, p):
    """one byte lane of add_mod_bytes: s = x + y (< 512), min(s, s - p) in uint32"""
    s = x + y
    return umin(s, (s - np.uint64(p)) & U32)


def sample(p, rng):
    top = (1 << 31) - 1
    v = [0, 1, -1, top, -top, top - 1, -top + 1]
    for end in (top, -top, 0):
        for base in (p, p // 2):
            m0 = end // base
            for m in range(m0 - 40, m0 + 41):
                for d in (-1, 0, 1):
                    v.append(m * base + d)
    v = np.array([x for x in v if -top <= x <= top], dtype=np.int64)
    return np.concatenate([v, rng.integers(-top, top + 1, 1 << 20, dtype=np.int64)])


def test_constants_keep_the_barrett_quotient_within_one():
    for p in MODULI:
        magic, off = host_constants(p)
        assert magic < 1 << 32 and 0 <= off < p and (off - (-(1 << 31))) % p == 0
        assert 0 <= (1 << 32) - magic * p < p                       # 2^32 / p - magic < 1: q undershoots floor(w / p) by <= 1


def test_plain_reduction_matches_python_mod():
    rng = np.random.default_rng(7)
    for p in MODULI:
        magic, off = host_constants(p)
        v = sample(p, rng)
        got = mod_s32(v, p, magic, off)
        edge = v.size - (1 << 20)                                   # the hand-picked values: Python integers
        assert [int(x) for x in got[:edge]] == [x % p for x in v[:edge].tolist()], p
        assert np.array_equal(got, (v % p).astype(np.uint64)), p    # numpy's % on int64 is Python's floor modulo
        assert int(got.max()) < p


def test_add_form_matches_python_mod():
    rng = np.random.default_rng(11)
    for p in MODULI:
        magic, off = host_constants(p)
        v = sample(p, rng)
        y = rng.integers(0, p, v.size).astype(np.uint64)           # the stored lower-half byte, in [0, p)
        y[:p] = np.arange(p, dtype=np.uint64)                       # every byte value at least once
        y[-p:] = np.arange(p, dtype=np.uint64)[::-1]
        got = add_mod_byte(mod_s32(v, p, magic, off), y, p)
        want = ((v % p) + y.astype(np.int64)) % p
        assert np.array_equal(got, want.astype(np.uint64)), p
        # the same as reducing v + y directly, which is what the fp64 epilogue did before the add moved after the reduction
        assert np.array_equal(got, ((v + y.astype(np.int64)) % p).astype(np.uint64)), p

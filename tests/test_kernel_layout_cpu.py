"""CPU re-derivation of the shared-memory layout claims of the fp64 DMMA kernel (matrel_b200/csrc/gemm_f64.cu, DESIGN 4.1):
the formulas are read from the source and checked exhaustively -- a wrong permutation or swizzle would still give correct
products (the tests on the GPU cannot see it) but would bring the bank conflicts back."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = open(os.path.join(ROOT, "matrel_b200", "csrc", "gemm_f64.cu")).read()


def c_expr(name):
    body = re.search(name + r"\(int (\w)\) \{ return ([^;]*); \}", SRC)
    var, expr = body.group(1), body.group(2)
    return lambda v: eval(expr, {}, {var: v})          # plain C integer expression with >>, &, +, *


kpos_of_k = c_expr("kpos_of_k")
k_of_kpos = c_expr("k_of_kpos")
BK = 16


def kset(s):                                            # k values of MMA step s, in thread-in-group order t = 0..3
    return [2 * s + (t & 1) + 8 * (t >> 1) for t in range(4)]


def test_ksets_partition_the_stage():
    assert "k_t = 2s + (t&1) + 8*(t>>1)" in SRC
    assert sorted(k for s in range(4) for k in kset(s)) == list(range(BK))


def test_padded_layout_permutation_makes_each_kset_four_consecutive_rows():
    assert sorted(kpos_of_k(k) for k in range(BK)) == list(range(BK))            # a permutation
    assert all(k_of_kpos(kpos_of_k(k)) == k for k in range(BK))                 # with the inverse the producer uses
    for s in range(4):
        assert [kpos_of_k(k) for k in kset(s)] == [4 * s, 4 * s + 1, 4 * s + 2, 4 * s + 3]


def test_swizzled_layout_gives_a_half_warp_16_distinct_8_byte_slots():
    """MODE_K tile: rows of 128 bytes (16 doubles of k), 16-byte chunk index ^= row & 7.  A half-warp of an m8n8k4 fragment
    load reads 4 consecutive rows x the 4 k of the step: all 16 accesses must fall into different 8-byte bank pairs."""
    for s in range(4):
        for row0 in range(0, 128, 4):                                           # half-warps start at multiples of 4 rows
            slots = set()
            for g in range(4):
                r = row0 + g
                for k in kset(s):
                    chunk = (k >> 1) ^ (r & 7)                                  # SWIZZLE_128B
                    slots.add(2 * chunk + (k & 1))                              # 8-byte slot inside the 128-byte row
            assert len(slots) == 16, (s, row0)


# ---- work-item order of the CTA-pair wgmma GEMM (matrel_b200/csrc/gemm_ozaki.cu, struct Oz2Items) ------------------------------
OZ_SRC = open(os.path.join(ROOT, "matrel_b200", "csrc", "gemm_ozaki.cu")).read()


def oz2_items(ksplit, npairs, ncl, cl, nmod, nk):
    """Python restatement of Oz2Items<KSPLIT>::next, statement by statement: (mi, t2, kc0, kcn, add) in execution order."""
    out = []
    if not ksplit:
        w = cl
        while w < npairs * nmod:
            mi = w // npairs
            out.append((mi, w - mi * npairs, 0, nk, False))
            w += ncl
        return out
    rot = npairs % ncl
    first_of = lambda mi: (cl + ncl - (mi * rot) % ncl) % ncl
    cur_mi, cur_kh, cur_t2 = 0, 0, first_of(0)
    while cur_mi < nmod:
        if cur_t2 < npairs:
            kcn = nk >> 1
            out.append((cur_mi, cur_t2, cur_kh * kcn, kcn, cur_kh != 0))
            cur_t2 += ncl
            continue
        if cur_kh == 0:
            cur_kh = 1
        else:
            cur_kh = 0
            cur_mi += 1
        cur_t2 = first_of(cur_mi)
    return out


def test_oz2_items_source_matches_the_restatement():
    """The formulas the restatement copies are the ones in the source (a changed kernel must change this test)."""
    for frag in ("return (cl + ncl - (mi * rot) % ncl) % ncl;", "rot(npairs_ % ncl_)", "if (w >= npairs * nmod) return false;",
                 "mi = w / npairs;", "t2 = w - mi * npairs;", "kcn = nk >> 1;", "kc0 = cur_kh * kcn;", "add = cur_kh != 0;",
                 "cur_t2 = first_of(cur_mi);"):
        assert frag in OZ_SRC, frag


def test_oz2_items_cover_every_item_once_and_keep_both_k_halves_on_one_cta_pair():
    """Default order: every (modulus, tile pair) exactly once over the CTA pairs, the whole K each.  K-split order: every (modulus,
    K half, tile pair) exactly once; both halves of a tile on the SAME CTA pair with the lower half first (the upper half's epilogue
    adds the byte the same thread stored -- no cross-CTA ordering exists to rely on); the load stays balanced although the
    leftover tile pairs of a sweep rotate over the CTA pairs."""
    for npairs, ncl, nmod, nk in [(2341, 74, 14, 128), (1755, 74, 14, 128), (2048, 74, 16, 128), (300, 74, 14, 64), (8, 74, 14, 8),
                                  (74, 74, 3, 2), (75, 37, 5, 16), (1, 1, 2, 4), (5, 3, 6, 10)]:
        flat = {}
        for cl in range(ncl):
            for (mi, t2, kc0, kcn, add) in oz2_items(False, npairs, ncl, cl, nmod, nk):
                assert (mi, t2) not in flat and (kc0, kcn, add) == (0, nk, False)
                flat[(mi, t2)] = cl
        assert len(flat) == npairs * nmod
        owner, loads = {}, []
        for cl in range(ncl):
            seq = oz2_items(True, npairs, ncl, cl, nmod, nk)
            loads.append(len(seq))
            pos = {}
            for i, (mi, t2, kc0, kcn, add) in enumerate(seq):
                kh = 1 if add else 0
                assert kcn == nk // 2 and kc0 == kh * kcn and (mi, kh, t2) not in owner
                owner[(mi, kh, t2)] = cl
                pos[(mi, kh, t2)] = i
            for (mi, kh, t2), i in pos.items():
                if kh == 1:
                    assert pos[(mi, 0, t2)] < i          # same CTA pair, lower half first
        assert len(owner) == 2 * npairs * nmod
        assert all(owner[(mi, 1 - kh, t2)] == cl for (mi, kh, t2), cl in owner.items())
        if npairs >= ncl:
            assert max(loads) - min(loads) <= 2 * (-(-nmod * (npairs % ncl) // ncl) - (nmod * (npairs % ncl)) // ncl) + 2

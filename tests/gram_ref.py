"""The triangular tile rule of the Ozaki-II Gram route (DESIGN section 4.1.2), restated from the elements each tile holds.

The engine's job buffer holds one slot of `slot_stride(blk)` lines per block row (rows) and block column (columns).  Output
block (i, j) of a Gram product sits at rows [s_i ss, s_i ss + m_i) and columns [s_j ss, s_j ss + m_j), s = compact slot, ss =
slot stride.  Its int8 GEMM runs in tiles of TM x TN buffer elements.  The route keeps, for every block on or above the block
diagonal, the tiles that hold an element of an upper block or an element on or above the diagonal of a diagonal block; with the
CTA-pair kernel (ss a multiple of 2 TM) tiles come in whole vertical pairs (2a, 2a + 1)."""
import numpy as np

TM, TN = 128, 256


def slot_stride(blk):
    return -(-blk // TM) * TM


def paired(blk):
    return slot_stride(blk) % (2 * TM) == 0


def _holds_upper(a, b, r0, c0, m, n, diag):
    """Tile (a, b) holds an element (r, c) of the m x n block at buffer (r0, c0) with r <= c (any element if not diag)."""
    rows = range(max(a * TM, r0), min(a * TM + TM, r0 + m))
    cols = range(max(b * TN, c0), min(b * TN + TN, c0 + n))
    if not rows or not cols:
        return False
    return not diag or rows[0] - r0 <= cols[-1] - c0  # its first row and last column decide


def block_tiles(rs, cs, m, n, blk, diag):
    """The tiles kept for output block (rs, cs) (compact slots) of m x n."""
    ss, pr = slot_stride(blk), paired(blk)
    r0, c0 = rs * ss, cs * ss
    a_lo, a_hi = r0 // TM, -(-(r0 + m) // TM)
    if pr:
        a_lo, a_hi = a_lo & ~1, a_hi + (a_hi & 1)
    kept = set()
    for a in range(a_lo, a_hi):
        for b in range(c0 // TN, -(-(c0 + n) // TN)):
            mates = (a, a ^ 1) if pr else (a,)
            if any(_holds_upper(x, b, r0, c0, m, n, diag) for x in mates):
                kept.add((a, b))
    return kept


def gram_tiles(dims, outputs, blk):
    """The tile set of a Gram product: dims[s] = order of slot s, outputs = (rs, cs) slot pairs of its output blocks."""
    tiles = set()
    for rs, cs in outputs:
        if rs <= cs:
            tiles |= block_tiles(rs, cs, dims[rs], dims[cs], blk, rs == cs)
    return tiles


def gram_int8_ops(dims, outputs, blk, T, K):
    """tc_int8_ops of the Gram route: kept tiles x moduli x 2 TM TN Kpad."""
    kpad = -(-K // 128) * 128
    return len(gram_tiles(dims, outputs, blk)) * T * 2 * TM * TN * kpad


def element_masks(dims, outputs, blk):
    """Buffer-sized masks: elements of upper blocks or on / above a diagonal block's diagonal; elements of any output block."""
    ss = slot_stride(blk)
    rows = len(dims) * ss
    cols = -(-rows // TN) * TN
    upper = np.zeros((rows, cols), dtype=bool)
    anyb = np.zeros((rows, cols), dtype=bool)
    for rs, cs in outputs:
        m, n = dims[rs], dims[cs]
        r0, c0 = rs * ss, cs * ss
        anyb[r0:r0 + m, c0:c0 + n] = True
        if rs < cs:
            upper[r0:r0 + m, c0:c0 + n] = True
        elif rs == cs:
            upper[r0:r0 + m, c0:c0 + n] = np.triu(np.ones((m, n), dtype=bool))
    return upper, anyb

"""The triangular tile rule of the Ozaki-II Gram route (tests/gram_ref.py), checked element by element without a GPU: every
element on or above the diagonal is in exactly one kept tile, no kept tile holds only elements below it, and CTA pairs stay
whole.  The GPU tests compare the engine's tc_int8_ops with the same rule."""
import numpy as np
import pytest

from tests.gram_ref import TM, TN, element_masks, gram_tiles, paired, slot_stride


def check_rule(dims, outputs, blk):
    tiles = gram_tiles(dims, outputs, blk)
    upper, anyb = element_masks(dims, outputs, blk)
    kept = np.zeros((upper.shape[0] // TM, upper.shape[1] // TN), dtype=bool)
    for a, b in tiles:
        kept[a, b] = True
    cover = np.repeat(np.repeat(kept, TM, axis=0), TN, axis=1)
    assert cover[upper].all()                                   # the tiles partition the buffer: covered means exactly once
    for a, b in tiles:
        t_any = anyb[a * TM:(a + 1) * TM, b * TN:(b + 1) * TN]
        t_up = upper[a * TM:(a + 1) * TM, b * TN:(b + 1) * TN]
        assert t_up.any() or not t_any.any(), (a, b)             # never wholly below the diagonal
        if not t_any.any():
            assert paired(blk) and (a ^ 1, b) in tiles         # a tile without elements is the padding half of a pair
    if paired(blk):
        assert all((a ^ 1, b) in tiles for a, b in tiles)
    return tiles


@pytest.mark.parametrize("blk", [64, 128, 256, 640, 1024])
@pytest.mark.parametrize("nb,last", [(1, None), (3, None), (4, 1), (5, 37), (6, -1)])
def test_rule_covers_the_upper_triangle_once(blk, nb, last):
    dims = [blk] * nb
    if last is not None:
        dims[-1] = blk - 1 if last == -1 else min(blk, last)
    outputs = [(i, j) for i in range(nb) for j in range(nb)]
    check_rule(dims, outputs, blk)


@pytest.mark.parametrize("blk", [256, 640, 1024])
def test_rule_with_absent_output_blocks(blk):
    dims = [blk, blk, blk, blk - 100]
    outputs = [(i, j) for i in range(4) for j in range(4) if (i, j) not in ((0, 2), (2, 0), (1, 3), (3, 1))]
    check_rule(dims, outputs, blk)


def test_tile_count_of_sixteen_blocks_of_1024():
    dims = [1024] * 16
    tiles = check_rule(dims, [(i, j) for i in range(16) for j in range(16)], 1024)
    assert len(tiles) == 120 * 32 + 16 * 20 == 4160


def test_slot_stride_and_pairing():
    assert [slot_stride(b) for b in (64, 200, 256, 640, 1024)] == [128, 256, 256, 640, 1024]
    assert [paired(b) for b in (64, 256, 640, 1024)] == [False, True, False, True]

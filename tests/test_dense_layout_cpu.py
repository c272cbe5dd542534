"""CPU tests of how MatfastSession.fromDense reads a 2-D array's strides: which dimension is contiguous and the leading
dimension it hands to mr_matrix_from_dense."""
import numpy as np
import pytest

from matrel_b200.dataset import _dense_layout


def _layout(a):
    return _dense_layout(a.shape, tuple(s // a.itemsize for s in a.strides))


def test_orders_and_slices():
    big = np.zeros((305, 207))
    assert _layout(big) == (1, 207)
    assert _layout(big.T) == (0, 207)
    assert _layout(big[2:302, 3:203]) == (1, 207)
    f = np.asfortranarray(big)
    assert _layout(f) == (0, 305)
    assert _layout(f[1:301, 2:202]) == (0, 305)


def test_a_single_line_is_contiguous_both_ways():
    assert _layout(np.zeros((1, 257))) == (1, 257)
    assert _layout(np.asfortranarray(np.zeros((1, 257)))) == (1, 257)
    assert _layout(np.zeros((257, 1))) == (1, 1)
    assert _layout(np.asfortranarray(np.zeros((257, 1)))) == (1, 1)
    assert _dense_layout((257, 1), (1, 300)) == (0, 257)
    assert _layout(np.zeros((305, 207))[5:9, 4:5]) == (1, 207)


@pytest.mark.parametrize("shape, strides", [((4, 4), (2, 8)), ((4, 4), (8, 2)), ((4, 4), (0, 1)), ((4, 4), (-4, 1)), ((4, 4), (1, 2))])
def test_no_unit_stride_dimension_is_refused(shape, strides):
    with pytest.raises(ValueError, match="one unit-stride dimension"):
        _dense_layout(shape, strides)

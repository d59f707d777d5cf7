"""Plans for detectors with more than 93 classes: the heads' output convolution runs as one or two 96-column tiles, so inference
plans accept anchors + classes up to 192 and report larger shapes as unsupported.  Plans are host-only objects (no GPU needed)."""
import ctypes

import pytest

import yfv2  # noqa: F401


def _plan(A, C, N=1, H=352, W=352):
    import yfv2_engine
    lib = yfv2_engine.lib()
    h = ctypes.c_void_p()
    rc = lib.yfv2_plan_create(ctypes.byref(h), 0, N, H, W, A, C, 0)
    return lib, h, rc


def _packed_bytes(A, C):
    lib, h, rc = _plan(A, C)
    assert rc == 0, (A, C, lib.yfv2_last_error())
    nb = ctypes.c_size_t()
    assert lib.yfv2_plan_packed_bytes(h, ctypes.byref(nb)) == 0
    assert lib.yfv2_plan_destroy(h) == 0
    return nb.value


@pytest.mark.parametrize("A,C", [(3, 93), (3, 94), (3, 150), (3, 189), (4, 188), (1, 191)])
def test_plans_up_to_two_output_tiles(A, C):
    counts = []
    for c in (80, C):                                                                   # the same launches as at 80 classes
        lib, h, rc = _plan(A, c)
        assert rc == 0, (A, c, lib.yfv2_last_error())
        n = ctypes.c_int()
        assert lib.yfv2_plan_forward_launches(h, ctypes.byref(n)) == 0
        counts.append(n.value)
        assert lib.yfv2_plan_destroy(h) == 0
    assert counts[0] == counts[1]


@pytest.mark.parametrize("A,C", [(3, 190), (8, 185)])
def test_more_than_two_tiles_is_unsupported(A, C):
    lib, h, rc = _plan(A, C)
    assert rc == -3                                                                     # YFV2_EUNSUPPORTED
    assert b"anchors+classes = %d" % (A + C) in lib.yfv2_last_error()


def test_packed_bytes_of_one_tile_shapes_are_unchanged():
    """The packed-weight layout of shapes that fit one tile is the one earlier builds used (values pinned from them)."""
    assert _packed_bytes(3, 80) == 1091616
    assert _packed_bytes(2, 20) == 1072672


def test_packed_bytes_grow_by_the_second_cls_tile():
    """Above 96 output columns each of the two cls heads packs a [192][72] folded matrix and bias instead of [96][72]; the reg heads
    (4A <= 32 columns) and everything else keep their size, apart from the [72][A+C] output-conv pack."""
    one, two = _packed_bytes(3, 93), _packed_bytes(3, 94)
    out_conv = 4 * (72 + 2) * 4                                                          # round4(97) - round4(96) = 4 columns
    assert two - one == 2 * 4 * (96 * 72 + 96) + out_conv
    assert _packed_bytes(3, 189) - two == 4 * (72 + 2) * (192 - 100)                     # only the output-conv pack widens further

"""Detection on regions of frames without a GPU: the cross-region merge's restatement (tests/region_oracle.py) on hand-built
cases, every refusal of yfv2_merge_regions before anything is launched, tile_regions' geometry and crop_frame's refusals."""
import ctypes
import math

import numpy as np
import pytest

import yfv2  # noqa: F401
import region_cases as rc
import region_oracle as ro

CASES = {c[0]: c for c in rc.hand_cases()}


def run(name):
    _, d, n, r, F, W, H, thr, metric, max_det = CASES[name]
    return ro.merge(d, n, r, F, W, H, thr, metric, max_det)


def confs(out, counts, f=0):
    return [float(v) for v in out[f, :counts[f], 4]]


@pytest.mark.parametrize("name,want", [("iou_seam_below_thr", [0.9]), ("iou_seam_at_thr", [0.9, 0.8]),
                                       ("ios_seam_thr_0.99", [0.9]), ("ios_seam_thr_1", [0.9, 0.8])])
def test_object_on_a_seam_just_above_and_below_the_threshold(name, want):
    out, counts, src = run(name)
    assert confs(out, counts) == pytest.approx(want)
    assert out[0, 0, :4].tolist() == [60.0, 20.0, 140.0, 120.0]                 # the full view, mapped with scale 2
    if len(want) == 2:
        assert out[0, 1, :4].tolist() == [60.0, 20.0, 100.0, 120.0] and src[0, :2].tolist() == [0, 1]


def test_same_region_rows_and_other_classes_are_never_suppressed():
    out, counts, src = run("same_region_and_other_class")
    # region 1's class-1 row (conf .6) is the only one a kept row of another region and the same class covers
    assert confs(out, counts) == pytest.approx([0.9, 0.8, 0.7]) and out[0, :3, 5].tolist() == [1.0, 1.0, 2.0]
    assert src[0, :4].tolist() == [0, 1, 2, -1]


def test_conf_ties_across_regions_go_by_region_then_row():
    out, counts, src = run("conf_ties")
    assert counts[0] == 2 and src[0, :2].tolist() == [0, 1]                     # region 0 row 0 wins; its twins are suppressed


def test_iou_exactly_at_the_threshold_is_not_suppressed():
    out, counts, _ = run("iou_exactly_half_thr_0.5")
    assert counts[0] == 2 and out[0, 1, :4].tolist() == [0.0, 0.0, 2.0, 3.0]
    out, counts, _ = run("iou_exactly_half_thr_%r" % float(np.nextafter(0.5, 0.0)))
    assert counts[0] == 1


@pytest.mark.parametrize("metric", [0, 1])
def test_thresholds_outside_zero_one(metric):
    # below 0 every same-class row of another region goes, disjoint or not; at 0 only overlapping ones; from 1 up none
    assert run("thr_-0.1_metric_%d" % metric)[1][0] == 2
    out, counts, src = run("thr_0_metric_%d" % metric)
    assert src[0, :3].tolist() == [0, 1, 3]
    for thr in ("1", "1.5"):
        assert run("thr_%s_metric_%d" % (thr, metric))[1][0] == 4


def test_degenerate_boxes_and_nan():
    out, counts, src = run("degenerate_metric_0")
    # the NaN-conf row (region 0 row 2) is dropped; zero-area and NaN boxes never suppress under IoU; -0 ties with +0 by region
    assert src[0, :6].tolist() == [0, 4, 1, 5, 7, 3]
    assert math.copysign(1.0, out[0, 5, 4]) == -1.0                             # conf copied exactly
    # IoS: the NaN area loses the min() to the other box's area, so the kept NaN box at .6 removes region 0's -0 row
    out, counts, src = run("degenerate_metric_1")
    assert src[0, :6].tolist() == [0, 4, 1, 5, 7, 6]


def test_empty_regions_and_frames_without_regions():
    out, counts, src = run("empty_regions_and_frames")
    assert counts.tolist() == [0, 1, 0, 0, 0] and out[1, 0, :4].tolist() == [60.0, 10.0, 100.0, 50.0] and src[1, 0] == 1
    assert not out[[0, 2, 3, 4]].any() and (src[[0, 2, 3, 4]] == -1).all()


def test_max_det_one():
    out, counts, src = run("max_det_1")
    assert counts[0] == 1 and out[0, 0, 4] == np.float32(0.95) and src[0, 0] == 1


def test_mapping_is_a_product_then_a_sum():
    rows = np.array([[0.1, 0.3, 351.9, 350.7, 0.5, 3.0]], np.float32)
    got = ro.map_rows(rows, (7, 11, 641, 479), 352, 352)[0]
    sx, sy = 641 / 352, 479 / 352
    want = [float(np.float32(0.1)) * sx + 7, float(np.float32(0.3)) * sy + 11, float(np.float32(351.9)) * sx + 7,
            float(np.float32(350.7)) * sy + 11]
    assert got[:4].tolist() == want and got[4] == np.float32(0.5) and got[5] == 3.0


# ---- yfv2_merge_regions refusals: checked on the host before any launch, so this runs without a GPU -------------------------------
def call(regions, T=None, F=2, W=352, H=352, mdi=300, max_det=300, thr=0.5, metric=1, dets=1, counts=1, out=1, oc=1):
    import yfv2_engine as eng
    L = eng.lib()
    arr = (eng.Region * max(len(regions), 1))(*[eng.Region(*r) for r in regions])
    T = len(regions) if T is None else T
    p = lambda v: ctypes.c_void_p(16) if v else None                         # never dereferenced: the checks come first
    rc_ = L.yfv2_merge_regions(p(dets), p(counts), arr if regions is not None else None, T, mdi, F, H, W, ctypes.c_double(thr),
                               metric, max_det, p(out), p(oc), None, None)
    return rc_, L.yfv2_last_error().decode()


GOOD = [(0, 0, 0, 100, 100), (0, 50, 0, 100, 100), (1, 0, 0, 10, 10)]


@pytest.mark.parametrize("kw,regs,msg", [
    (dict(dets=0), GOOD, "null"), (dict(counts=0), GOOD, "null"), (dict(out=0), GOOD, "null"), (dict(oc=0), GOOD, "null"),
    (dict(T=0), GOOD, "T, F, W, H"), (dict(F=0), GOOD, "T, F, W, H"), (dict(W=0), GOOD, "T, F, W, H"), (dict(H=0), GOOD, "T, F, W, H"),
    (dict(mdi=0), GOOD, "max_det_in"), (dict(mdi=4097), GOOD, "max_det_in"), (dict(max_det=0), GOOD, "max_det"),
    (dict(max_det=4097), GOOD, "max_det"), (dict(metric=2), GOOD, "metric"), (dict(metric=-1), GOOD, "metric"),
    (dict(thr=float("nan")), GOOD, "NaN"),
    (dict(), [(0, 0, 0, 0, 100)], "region 0: w and h"), (dict(), [(0, 0, 0, 100, 100), (0, 0, 0, 100, 0)], "region 1: w and h"),
    (dict(), [(0, -1, 0, 100, 100)], "region 0: x0 and y0"), (dict(), [(0, 0, -2, 100, 100)], "region 0: x0 and y0"),
    (dict(), [(2, 0, 0, 100, 100)], "region 0: frame outside"), (dict(), [(-1, 0, 0, 100, 100)], "region 0: frame outside"),
    (dict(), [(1, 0, 0, 10, 10), (0, 0, 0, 10, 10)], "region 1: frame index decreases"),
    (dict(mdi=300), [(0, 0, 0, 10, 10)] * 28, "region 27: frame 0 has 28 regions"),
    (dict(mdi=8), [(0, 0, 0, 10, 10)] * 1025, "region 1024: frame 0 has 1025 regions"),
    (dict(mdi=4096), [(0, 0, 0, 10, 10)] * 524288, "2^31"),
])
def test_merge_regions_refusals_before_any_launch(kw, regs, msg):
    rc_, err = call(regs, **kw)
    assert rc_ == -1 and msg in err, (rc_, err)


def test_the_limits_themselves_pass_the_checks():
    """27 regions of 300 rows, 2 of 4096 and 1024 of 8 are within the limits: the call gets past every check and only then fails,
    with YFV2_ECUDA here for want of a device (on a GPU machine these would be real launches: not done with fake pointers)."""
    pytest.importorskip("torch")
    import torch
    if torch.cuda.is_available():
        pytest.skip("the launch would read the fake pointers")
    for mdi, k in ((300, 27), (4096, 2), (8, 1024)):
        rc_, err = call([(0, 0, 0, 10, 10)] * k, mdi=mdi)
        assert rc_ == -2, (mdi, k, err)


# ---- tile_regions ----------------------------------------------------------------------------------------------------------------
def covered(w, h, tiles):
    m = np.zeros((h, w), bool)
    for x0, y0, tw, th in tiles:
        m[y0:y0 + th, x0:x0 + tw] = True
    return m.all()


@pytest.mark.parametrize("w,h,cols,rows,overlap,layout", [
    (1920, 1080, 3, 2, 0.2, "bgr"), (1920, 1080, 3, 2, 0.2, "nv12"), (1921, 1081, 4, 3, 0.25, "bgr"), (1922, 1081, 3, 3, 0.1, "yuyv"),
    (1278, 718, 5, 4, 0.3, "i420"), (640, 480, 2, 2, 0.0, "rgb"), (37, 29, 6, 5, 0.5, "gray"), (2, 2, 3, 3, 0.2, "nv21"),
    (1, 1, 2, 2, 0.2, "bgr"), (1000, 10, 7, 1, 0.2, "uyvy")])
def test_tile_geometry(w, h, cols, rows, overlap, layout):
    from utils.frames import tile_regions
    tiles = tile_regions(w, h, cols, rows, overlap, full_frame=True, layout=layout)
    assert tiles[0] == (0, 0, w, h) and len(tiles) == 1 + cols * rows
    tiles = tiles[1:]
    assert covered(w, h, tiles)
    tw, th = tiles[0][2], tiles[0][3]
    xs = sorted({t[0] for t in tiles})
    ys = sorted({t[1] for t in tiles})
    assert xs[-1] + tw == w and ys[-1] + th == h and xs[0] == 0 and ys[0] == 0        # the last tile ends on the edge
    for x0, y0, a, b in tiles:
        assert (a, b) == (tw, th) and 0 <= x0 and x0 + a <= w and 0 <= y0 and y0 + b <= h
    for v, size, k in ((xs, tw, cols), (ys, th, rows)):
        for p, q in zip(v, v[1:]):
            assert p + size - q >= overlap * size - 2                                    # adjacent tiles overlap
    if layout in ("nv12", "nv21", "i420", "yv12"):
        assert all(v % 2 == 0 for t in tiles for v in t)
    if layout in ("yuyv", "uyvy", "yvyu"):
        assert all(t[0] % 2 == 0 and t[2] % 2 == 0 for t in tiles)


def test_one_tile_without_the_full_frame_is_the_frame():
    from utils.frames import tile_regions
    assert tile_regions(1920, 1080, 1, 1, 0.2, full_frame=False) == [(0, 0, 1920, 1080)]
    assert tile_regions(1920, 1080, 1, 1, 0.2) == [(0, 0, 1920, 1080)] * 2
    with pytest.raises(ValueError):
        tile_regions(1920, 1080, 0, 1)


# ---- crop_frame refusals ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout,shape,window,msg", [
    ("bgr", (100, 120, 3), (0, 0, 121, 10), "not inside"), ("bgr", (100, 120, 3), (-1, 0, 10, 10), "not inside"),
    ("bgr", (100, 120, 3), (0, 0, 0, 10), "not inside"), ("gray", (100, 120), (0, 95, 10, 6), "not inside"),
    ("rgb_chw", (3, 100, 120), (110, 0, 11, 10), "not inside"), ("nv12", (150, 120), (1, 0, 10, 10), "even"),
    ("i420", (150, 120), (0, 0, 10, 11), "even"), ("yv12", (150, 120), (0, 3, 10, 10), "even"),
    ("yuyv", (100, 120, 2), (1, 0, 10, 10), "even x0 and w"), ("uyvy", (100, 120, 2), (0, 0, 11, 10), "even x0 and w"),
    ("bgr", (100, 120, 4), (0, 0, 10, 10), "bgr"), ("nope", (100, 120, 3), (0, 0, 10, 10), "layout"),
])
def test_crop_frame_refusals(layout, shape, window, msg):
    import yfv2_engine as eng
    with pytest.raises(eng.Yfv2Error, match=msg):
        eng.crop_frame(np.zeros(shape, np.uint8), layout, *window)


def test_crop_frame_returns_views():
    import torch
    import yfv2_engine as eng
    f = np.arange(100 * 120 * 3, dtype=np.uint32).astype(np.uint8).reshape(100, 120, 3)
    c = eng.crop_frame(f, "bgr", 10, 20, 30, 40)
    assert c.shape == (40, 30, 3) and np.shares_memory(c, f) and np.array_equal(c, f[20:60, 10:40])
    buf = torch.zeros((150, 120), dtype=torch.uint8)
    y, uv = eng.crop_frame(buf, "nv12", 10, 20, 30, 40)
    assert y.shape == (40, 30) and uv.shape == (20, 30) and y.data_ptr() == buf[20:, 10:].data_ptr()
    assert uv.data_ptr() == buf[100 + 10:, 10:].data_ptr()
    y, u, v = eng.crop_frame(buf, "i420", 10, 20, 30, 40)
    assert u.shape == v.shape == (20, 15)
    assert u.data_ptr() == buf.reshape(-1)[100 * 120 + 10 * 60 + 5:].data_ptr()
    assert v.data_ptr() == buf.reshape(-1)[100 * 120 + 50 * 60 + 10 * 60 + 5:].data_ptr()

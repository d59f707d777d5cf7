"""Greedy non-maximum merging of the cross-region merge without a GPU: tests/region_nmm_oracle.py on hand-built cases
(tests/region_nmm_cases.py), every refusal of yfv2_merge_regions_nmm before anything is launched, and the mode / want_merged /
merge_mode checks of the Python API."""
import ctypes
import math

import numpy as np
import pytest

import yfv2  # noqa: F401
import region_cases as rc
import region_nmm_cases as nc
import region_nmm_oracle as rno
import region_oracle as ro

CASES = {c[0]: c for c in nc.all_hand_cases()}


def run(name):
    return rno.merge_nmm(*CASES[name][1:])


def boxes(out, counts, f=0):
    return out[f, :counts[f], :4].tolist()


@pytest.mark.parametrize("name", sorted(CASES))
def test_rows_counts_and_sources_are_the_nms_merge(name):
    """Only the four box columns may differ from yfv2_merge_regions; each NMM box contains the NMS box (or carries NaN)."""
    out, counts, src, merged = run(name)
    wo, wc, ws = ro.merge(*CASES[name][1:])
    assert np.array_equal(counts, wc) and np.array_equal(src, ws)
    assert np.array_equal(out[..., 4:].view(np.uint64), wo[..., 4:].view(np.uint64))
    for f in range(len(counts)):
        n = counts[f]
        a, b = out[f, :n, :4], wo[f, :n, :4]
        with np.errstate(invalid="ignore"):
            inside = (a[:, :2] <= b[:, :2]).all(1) & (a[:, 2:] >= b[:, 2:]).all(1)
        assert (inside | np.isnan(a).any(1) | np.isnan(b).any(1)).all(), (name, f)
        assert (merged[f, n:] == 0).all() and not out[f, n:].any()
        assert ((merged[f, :n] == 0) <= (a == b).all(1) | np.isnan(b).any(1)).all()   # an untouched box is the NMS box


def test_a_higher_scoring_piece_absorbs_the_whole_box():
    out, counts, src, merged = run("piece_absorbs_whole")
    assert counts[0] == 1 and src[0, 0] == 1 and out[0, 0, 4] == np.float32(0.95)           # the piece stays the winner
    assert boxes(out, counts) == [[60.0, 20.0, 140.0, 120.0]] and merged[0, 0] == 1
    assert ro.merge(*CASES["piece_absorbs_whole"][1:])[0][0, 0, :4].tolist() == [60.0, 20.0, 100.0, 120.0]


def test_two_overlapping_pieces_make_one_box():
    out, counts, _, merged = run("two_pieces")
    assert boxes(out, counts) == [[60.0, 20.0, 140.0, 60.0]] and merged[0, 0] == 1


def test_the_recheck_is_against_the_grown_box():
    out, counts, _, merged = run("chain_grows")
    assert boxes(out, counts) == [[0.0, 0.0, 10.0, 4.0]] and merged[0, 0] == 2
    out, counts, _, merged = run("chain_rejects")
    # against box_i the last row would fold (IoS 1) and give 0..16 x 0..12; against B it has IoS 1/3
    assert boxes(out, counts) == [[0.0, 0.0, 16.0, 4.0]] and merged[0, 0] == 1


@pytest.mark.parametrize("metric,grown", [("iou", [0.0, 0.0, 6.0, 4.0]), ("ios", [0.0, 0.0, 16.0, 8.0])])
def test_overlap_exactly_at_the_threshold_does_not_fold(metric, grown):
    out, counts, _, merged = run("%s_exactly_thr_at" % metric)
    assert merged[0, 0] == 1 and out[0, 0, 3] == 4.0 and out[0, 0, 2] == (6.0 if metric == "iou" else 16.0)
    out, counts, _, merged = run("%s_exactly_thr_below" % metric)
    assert merged[0, 0] == 2 and boxes(out, counts) == [grown]


def test_a_row_goes_to_the_first_output_row_that_matches_it():
    out, counts, _, merged = run("first_of_two_matches")
    assert boxes(out, counts) == [[0.0, 0.0, 13.0, 10.0], [8.0, 0.0, 18.0, 10.0]] and merged[0, :2].tolist() == [1, 0]


@pytest.mark.parametrize("max_det", [1, 10])
def test_same_region_and_other_class_rows_never_merge(max_det):
    out, counts, _, merged = run("same_region_and_other_class_max_det_%d" % max_det)
    assert out[0, 0, :4].tolist() == [10.0, 10.0, 50.0, 50.0] and not merged.any()
    assert counts[0] == (1 if max_det == 1 else 3)


def test_nan_boxes():
    out, counts, src, merged = run("nan_boxes_metric_0")
    # IoU: NaN overlaps never match; the finite rows fold into their output rows
    assert src[0, :4].tolist() == [0, 1, 2, 3] and merged[0, :4].tolist() == [1, 0, 0, 1]
    assert out[0, 0, :4].tolist() == [0.0, 0.0, 12.0, 10.0] and math.isnan(out[0, 1, 3]) and math.isnan(out[0, 2, 0])
    out, counts, src, merged = run("nan_boxes_metric_1")
    # IoS: the box with a NaN y2 absorbs both 30..40 rows; its NaN gives way to the first row's 40
    assert src[0, :3].tolist() == [0, 1, 2] and merged[0, :3].tolist() == [1, 2, 0]
    assert out[0, 1, :4].tolist() == [30.0, 30.0, 42.0, 40.0]


def test_rows_after_the_cap():
    out, counts, src, merged = run("max_det_1_rows_after_the_cap")
    # the row whose first suppressor is past the cap (52..62) belongs to no output row; 0..12 folds into the output row
    assert counts[0] == 1 and src[0, 0] == 0 and boxes(out, counts) == [[0.0, 0.0, 12.0, 10.0]] and merged[0, 0] == 1
    out, counts, src, merged = run("max_det_1")
    assert boxes(out, counts) == [[60.0, 20.0, 140.0, 120.0]] and merged[0, 0] == 1


def test_frames_are_independent():
    out, counts, src, merged = run("frames_and_scales")
    assert counts.tolist() == [1, 0, 1, 0] and merged[:, 0].tolist() == [1, 0, 1, 0]
    assert boxes(out, counts, 0) == boxes(out, counts, 2) == [[60.0, 20.0, 140.0, 120.0]]
    assert out[0, 0, 4] == np.float32(0.95) and out[2, 0, 4] == np.float32(0.9)


# ---- yfv2_merge_regions_nmm refusals: the checks of yfv2_merge_regions, named for the new call, before any launch ----------------
def call(regions, T=None, F=2, W=352, H=352, mdi=300, max_det=300, thr=0.5, metric=1, dets=1, counts=1, out=1, oc=1, merged=1):
    import yfv2_engine as eng
    L = eng.lib()
    arr = (eng.Region * max(len(regions), 1))(*[eng.Region(*r) for r in regions])
    T = len(regions) if T is None else T
    p = lambda v: ctypes.c_void_p(16) if v else None                         # never dereferenced: the checks come first
    rc_ = L.yfv2_merge_regions_nmm(p(dets), p(counts), arr, T, mdi, F, H, W, ctypes.c_double(thr), metric, max_det, p(out), p(oc),
                                   None, p(merged), None)
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
def test_merge_regions_nmm_refusals_before_any_launch(kw, regs, msg):
    rc_, err = call(regs, **kw)
    assert rc_ == -1 and err.startswith("merge_regions_nmm: ") and msg in err, (rc_, err)


def test_the_limits_themselves_pass_the_checks():
    """The limits of yfv2_merge_regions, with and without `merged`: past every check, then YFV2_ECUDA for want of a device."""
    pytest.importorskip("torch")
    import torch
    if torch.cuda.is_available():
        pytest.skip("the launch would read the fake pointers")
    for mdi, k in ((300, 27), (4096, 2), (8, 1024)):
        for merged in (0, 1):
            rc_, err = call([(0, 0, 0, 10, 10)] * k, mdi=mdi, max_det=4096, merged=merged)
            assert rc_ == -2, (mdi, k, err)


# ---- the Python API -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw,msg", [(dict(mode="wbf"), "mode must be 'nms' or 'nmm'"), (dict(mode="NMM"), "mode must be"),
                                    (dict(mode=None), "mode must be"), (dict(want_merged=True), "want_merged needs mode='nmm'")])
def test_merge_regions_mode_checks_come_first(kw, msg):
    """Refused before anything is looked at or copied: the tensors here are not even CUDA tensors."""
    import torch
    import yfv2_engine as eng
    with pytest.raises(eng.Yfv2Error, match=msg):
        eng.merge_regions(torch.zeros((1, 4, 6)), torch.zeros(1, dtype=torch.int32), [(0, 0, 0, 10, 10)], 1, 352, 352, 0.5, "ios",
                          10, **kw)


def test_detect_regions_merge_mode_check_comes_first():
    import yfv2_engine as eng
    from utils import frames as uf
    with pytest.raises(eng.Yfv2Error, match="merge_mode must be 'nms' or 'nmm'"):
        uf.detect_regions(None, [np.zeros((8, 8, 3), np.uint8)], {"width": 352, "height": 352}, [[(0, 0, 8, 8)]], merge_mode="x")
    with pytest.raises(eng.Yfv2Error, match="merge_mode"):
        uf.detect_tiled(None, [np.zeros((8, 8, 3), np.uint8)], {"width": 352, "height": 352}, 1, 1, merge_mode="greedy")


def test_the_defaults_are_the_nms_merge():
    import inspect
    import yfv2_engine as eng
    from utils import frames as uf
    assert inspect.signature(eng.merge_regions).parameters["mode"].default == "nms"
    assert inspect.signature(eng.merge_regions).parameters["want_merged"].default is False
    assert inspect.signature(uf.detect_regions).parameters["merge_mode"].default == "nms"

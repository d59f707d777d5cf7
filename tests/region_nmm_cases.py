"""Hand-built inputs of yfv2_merge_regions_nmm (greedy non-maximum merging), shared by tests/test_regions_nmm_cpu.py (against the
expected boxes) and tests/test_regions_nmm_gpu.py (the kernel against tests/region_nmm_oracle.py).  Same layout as
tests/region_cases.py: (name, dets float32 [T, max_det_in, 6], counts int32 [T], regions [(frame, x0, y0, w, h)], F, W, H, thr,
metric, max_det).  Regions are 100 x 100 at scale 1 unless stated, so boxes are in frame pixels as written."""
import numpy as np

import region_cases as rc

TILE = (0, 0, 100, 100)


def hand_cases():
    c = []
    W = H = 100
    # a tile piece (x 60..100, conf .95) scoring above the full view's whole box (x 60..140, conf .9): IoS 1 keeps the piece and
    # suppresses the whole box; NMM grows the piece into it
    d, n, r = rc.pack([rc.seam(0.95)])
    c.append(("piece_absorbs_whole", d, n, r, 1, W, H, 0.5, 1, 10))
    # two pieces of one object from neighbouring tiles, overlapping each other (IoS .75), no whole box anywhere
    d, n, r = rc.pack([[(TILE, [(60.0, 20.0, 100.0, 60.0, 0.95, 0.0)]), (TILE, [(70.0, 20.0, 140.0, 60.0, 0.9, 0.0)])]])
    c.append(("two_pieces", d, n, r, 1, W, H, 0.5, 1, 10))
    # a chain: box_i (x 0..4) absorbs rows x 0..6 and x 2..10 (IoU 2/3 and 1/5 against box_i, thr .15); the grown B (x 0..6)
    # takes x 2..10 at IoU 2/5, and the last B is x 0..10
    d, n, r = rc.pack([[(TILE, [(0.0, 0.0, 4.0, 4.0, 0.9, 0.0)]), (TILE, [(0.0, 0.0, 6.0, 4.0, 0.8, 0.0)]),
                        (TILE, [(2.0, 0.0, 10.0, 4.0, 0.7, 0.0)])]])
    c.append(("chain_grows", d, n, r, 1, W, H, 0.15, 0, 10))
    # a chain where the grown B rejects a row box_i matched: box_i 0..4 x 0..4, row 0..16 x 0..4 (IoS 1) grows B to 0..16; row
    # 0..4 x 0..12 (IoS 1 against box_i) has IoS 16 / 48 = 1/3 against B
    d, n, r = rc.pack([[(TILE, [(0.0, 0.0, 4.0, 4.0, 0.9, 0.0)]), (TILE, [(0.0, 0.0, 16.0, 4.0, 0.8, 0.0)]),
                        (TILE, [(0.0, 0.0, 4.0, 12.0, 0.7, 0.0)])]])
    c.append(("chain_rejects", d, n, r, 1, W, H, 0.5, 1, 10))
    # overlap exactly at thr against the grown B, from dyadic corners.  IoU: box_i 0..4 x 0..4, row 0..6 x 0..4 (IoU 2/3) grows B
    # to area 24; row 0..4 x 0..3 (IoU 3/4 against box_i) has IoU 12 / 24 = 0.5 against B.  IoS: row 0..16 x 0..4 grows B to
    # area 64; row 0..4 x 0..8 has IoS 16 / 32 = 0.5 against B.  At thr 0.5 the last row does not fold, just below it does.
    iou = rc.pack([[(TILE, [(0.0, 0.0, 4.0, 4.0, 0.9, 0.0)]), (TILE, [(0.0, 0.0, 6.0, 4.0, 0.8, 0.0)]),
                    (TILE, [(0.0, 0.0, 4.0, 3.0, 0.7, 0.0)])]])
    ios = rc.pack([[(TILE, [(0.0, 0.0, 4.0, 4.0, 0.9, 0.0)]), (TILE, [(0.0, 0.0, 16.0, 4.0, 0.8, 0.0)]),
                    (TILE, [(0.0, 0.0, 4.0, 8.0, 0.7, 0.0)])]])
    for thr, tag in ((0.5, "at"), (float(np.nextafter(0.5, 0.0)), "below")):
        c.append(("iou_exactly_thr_%s" % tag,) + iou + (1, W, H, thr, 0, 10))
        c.append(("ios_exactly_thr_%s" % tag,) + ios + (1, W, H, thr, 1, 10))
    # a row two output rows match goes to the first: boxes 0..10 (.9) and 8..18 (.85) are both kept (IoS .2), the row 5..13
    # (IoS .625 with each) grows the first
    d, n, r = rc.pack([[(TILE, [(0.0, 0.0, 10.0, 10.0, 0.9, 0.0)]), (TILE, [(8.0, 0.0, 18.0, 10.0, 0.85, 0.0)]),
                        (TILE, [(5.0, 0.0, 13.0, 10.0, 0.8, 0.0)])]])
    c.append(("first_of_two_matches", d, n, r, 1, W, H, 0.5, 1, 10))
    # rows of the same region and rows of another class never merge, after the cap or not
    box = (10.0, 10.0, 50.0, 50.0)
    for max_det in (1, 10):
        d, n, r = rc.pack([[(TILE, [box + (0.9, 0.0), (10.0, 10.0, 60.0, 50.0, 0.8, 0.0)]), (TILE, [(10.0, 10.0, 55.0, 50.0, 0.7, 1.0)])]])
        c.append(("same_region_and_other_class_max_det_%d" % max_det, d, n, r, 1, W, H, 0.5, 1, max_det))
    # NaN corners: a NaN overlap neither suppresses nor folds under IoU; under IoS a NaN area loses min() to the other area, so a
    # row with a NaN corner can be absorbed and fold.  mn / mx return the row's value when a compare fails, so a NaN corner of B
    # gives way to the row's and a NaN corner of the row replaces B's
    d, n, r = rc.pack([[(TILE, [(0.0, 0.0, 10.0, 10.0, 0.9, 0.0), (30.0, 30.0, 40.0, float("nan"), 0.85, 0.0)]),
                        (TILE, [(float("nan"), 0.0, 10.0, 10.0, 0.8, 0.0), (30.0, 30.0, 40.0, 40.0, 0.75, 0.0)]),
                        (TILE, [(0.0, 0.0, 12.0, 10.0, 0.7, 0.0), (30.0, 30.0, 42.0, 40.0, 0.6, 0.0)])]])
    for metric in (0, 1):
        c.append(("nan_boxes_metric_%d" % metric, d, n, r, 1, W, H, 0.5, metric, 10))
    # max_det 1 and rows after the cap: row (50..60, .8) would be kept next without the cap; row 52..62 (.7) matches only it, its
    # first suppressor beyond the cap, so it belongs to no output row; row 0..12 (.6) matches the output row and grows it
    d, n, r = rc.pack([[(TILE, [(0.0, 0.0, 10.0, 10.0, 0.9, 0.0)]), (TILE, [(50.0, 50.0, 60.0, 60.0, 0.8, 0.0), (0.0, 0.0, 12.0, 10.0, 0.6, 0.0)]),
                        (TILE, [(52.0, 50.0, 62.0, 60.0, 0.7, 0.0)])]])
    c.append(("max_det_1_rows_after_the_cap", d, n, r, 1, W, H, 0.5, 1, 1))
    # several frames, scale 2 for the full view, empty frames between
    d, n, r = rc.pack([rc.seam(0.95), [], rc.seam(0.85), [(TILE, [])]])
    c.append(("frames_and_scales", d, n, r, 4, W, H, 0.5, 1, 10))
    return c


def all_hand_cases():
    """These and tests/region_cases.py's hand cases (every NMS case is an NMM case too)."""
    return hand_cases() + rc.hand_cases()

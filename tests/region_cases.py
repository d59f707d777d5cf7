"""Hand-built and seeded inputs of yfv2_merge_regions, shared by tests/test_regions_cpu.py (against the expected rows) and
tests/test_regions_gpu.py (the kernel against tests/region_oracle.py).  Each case is (name, dets float32 [T, max_det_in, 6], counts
int32 [T], regions [(frame, x0, y0, w, h)], F, W, H, thr, metric, max_det)."""
import numpy as np

NAN = float("nan")


def pack(frames_regions, W=100, H=100, max_det_in=None):
    """frames_regions: per frame a list of (region (x0, y0, w, h), rows [(x1, y1, x2, y2, conf, cls), ...]).  Returns (dets, counts,
    regions); unused rows past a region's count hold garbage, which the merge must not read."""
    regs, blocks = [], []
    for f, lst in enumerate(frames_regions):
        for region, rows in lst:
            regs.append((f,) + tuple(region))
            blocks.append(rows)
    mdi = max_det_in or max([len(b) for b in blocks] + [1])
    dets = np.full((max(len(blocks), 1), mdi, 6), 7.0, np.float32)
    counts = np.zeros(max(len(blocks), 1), np.int32)
    for t, rows in enumerate(blocks):
        if rows:
            dets[t, :len(rows)] = np.asarray(rows, np.float32)
        counts[t] = len(rows)
    return dets, counts, regs


def seam(conf2):
    """A person cut by the seam of two 100-px tiles of a 200 x 100 frame (W = H = 100, scale 1): the left tile sees x 60..100, the
    full view (region 0, scale 2) the whole box x 60..140.  IoS of the fragment with the whole box is 1, IoU 0.5."""
    full = ((0, 0, 200, 200), [(30.0, 10.0, 70.0, 60.0, 0.9, 0.0)])             # x 60..140, y 20..120 in the frame
    left = ((0, 0, 100, 100), [(60.0, 20.0, 100.0, 120.0, conf2, 0.0)])
    return [full, left]


def hand_cases():
    c = []
    W = H = 100
    for thr, name in ((0.49, "iou_seam_below_thr"), (0.5, "iou_seam_at_thr")):
        d, n, r = pack([seam(0.8)])
        c.append((name, d, n, r, 1, W, H, thr, 0, 10))
    for thr in (0.99, 1.0):
        d, n, r = pack([seam(0.8)])
        c.append(("ios_seam_thr_%g" % thr, d, n, r, 1, W, H, thr, 1, 10))
    # rows of one region overlap fully and are never suppressed; another class is never suppressed
    box = (10.0, 10.0, 50.0, 50.0)
    d, n, r = pack([[((0, 0, 100, 100), [box + (0.9, 1.0), box + (0.8, 1.0)]),
                     ((0, 0, 100, 100), [box + (0.7, 2.0), box + (0.6, 1.0)])]])
    c.append(("same_region_and_other_class", d, n, r, 1, W, H, 0.5, 0, 10))
    # conf ties across regions: ordered by region, then by row
    d, n, r = pack([[((0, 0, 100, 100), [box + (0.5, 0.0), (60.0, 60.0, 70.0, 70.0, 0.5, 0.0)]),
                     ((0, 0, 100, 100), [box + (0.5, 0.0)]), ((0, 0, 100, 100), [box + (0.5, 0.0)])]])
    c.append(("conf_ties", d, n, r, 1, W, H, 0.5, 0, 10))
    # IoU exactly 0.5 in fp64 from dyadic corners with sx = 1 and sx = 2: not suppressed at 0.5, suppressed below
    d, n, r = pack([[((0, 0, 100, 100), [(0.0, 0.0, 4.0, 3.0, 0.9, 0.0)]),
                     ((0, 0, 200, 200), [(0.0, 0.0, 1.0, 1.5, 0.8, 0.0)])]])      # -> (0, 0, 2, 3): inter 6, union 12
    for thr in (0.5, np.nextafter(0.5, 0.0)):
        c.append(("iou_exactly_half_thr_%r" % float(thr), d, n, r, 1, W, H, float(thr), 0, 10))
    for thr in (-0.1, 0.0, 1.0, 1.5):
        for metric in (0, 1):
            d, n, r = pack([[((0, 0, 100, 100), [box + (0.9, 0.0), (60.0, 60.0, 70.0, 70.0, 0.8, 0.0)]),
                             ((0, 0, 100, 100), [box + (0.7, 0.0), (80.0, 80.0, 90.0, 90.0, 0.6, 0.0)])]])
            c.append(("thr_%g_metric_%d" % (thr, metric), d, n, r, 1, W, H, thr, metric, 10))
    # zero-area and NaN boxes, a NaN conf, -0 conf
    d, n, r = pack([[((0, 0, 100, 100), [(5.0, 5.0, 5.0, 9.0, 0.9, 0.0), (NAN, 1.0, 2.0, 3.0, 0.8, 0.0), (1.0, 1.0, 9.0, 9.0, NAN, 0.0),
                                         (1.0, 1.0, 9.0, 9.0, -0.0, 0.0)]),
                     ((0, 0, 100, 100), [(5.0, 5.0, 5.0, 9.0, 0.85, 0.0), (NAN, 1.0, 2.0, 3.0, 0.7, 0.0), (1.0, 1.0, 9.0, 9.0, 0.0, 0.0),
                                         (1.0, NAN, 9.0, 9.0, 0.6, 0.0)])]])
    for metric in (0, 1):
        c.append(("degenerate_metric_%d" % metric, d, n, r, 1, W, H, 0.1, metric, 10))
    # empty regions and frames without regions (frames 0, 2 and 4 have none)
    d, n, r = pack([[], [((0, 0, 100, 100), []), ((50, 0, 100, 100), [box + (0.9, 0.0)])], [], [((10, 10, 30, 30), [])], []])
    c.append(("empty_regions_and_frames", d, n, r, 5, W, H, 0.5, 1, 10))
    # max_det 1
    d, n, r = pack([seam(0.95)])
    c.append(("max_det_1", d, n, r, 1, W, H, 0.5, 1, 1))
    return c


def random_case(seed, F=300, max_regions=27, max_det_in=300, max_rows=40, classes=3, W=352, H=352, dense=False):
    """Seeded rows over F frames with 0..max_regions regions each: boxes on a coarse grid (many exact overlaps and ties), a few
    classes, conf quantised to 1/64 (many ties).  dense: every region of every frame has max_regions regions of max_det_in rows."""
    rs = np.random.RandomState(seed)
    regs = []
    for f in range(F):
        k = max_regions if dense else rs.randint(0, max_regions + 1)
        for _ in range(k):
            w, h = rs.randint(1, 1921), rs.randint(1, 1081)
            regs.append((f, rs.randint(0, 1920), rs.randint(0, 1080), w, h))
    T = max(len(regs), 1)
    dets = np.zeros((T, max_det_in, 6), np.float32)
    xy = rs.randint(0, 12, (T, max_det_in, 2)).astype(np.float32) * np.float32(W / 12)
    wh = rs.randint(1, 8, (T, max_det_in, 2)).astype(np.float32) * np.float32(W / 16)
    dets[..., 0:2], dets[..., 2:4] = xy, xy + wh
    dets[..., 4] = rs.randint(1, 65, (T, max_det_in)).astype(np.float32) / 64
    dets[..., 5] = rs.randint(0, classes, (T, max_det_in))
    counts = (np.full(T, max_det_in) if dense else rs.randint(0, max_rows + 1, T)).astype(np.int32)
    return dets, counts, regs

"""Hand-built inputs for the true-positive marking of get_batch_statistics (utils/utils.py:184-230), one per rule it follows.

Each builder returns a dict: outs (per image a float32 [n_i,6] array of NMS rows (x1, y1, x2, y2, conf, cls) by descending
conf), targets (float32 [nt,6] rows (image, class, x1, y1, x2, y2) in pixels), thr (the IoU threshold) and, for the small
cases, expect (the flags the rule gives, per image) so that the oracle itself is checked against the rule.  Everything is
numpy; nothing needs a GPU.
"""
import numpy as np

import synth

f32 = np.float32
NAN, INF = float("nan"), float("inf")


def rows(*r):
    return np.array(r, f32).reshape(-1, 6)


def det(x1, y1, x2, y2, cls=0, conf=0.5):
    return (x1, y1, x2, y2, conf, cls)


def tgt(img, x1, y1, x2, y2, cls=0):
    return (img, cls, x1, y1, x2, y2)


def filler(img, k, cls=3):
    """k annotations of image `img`, far from every box the cases test with."""
    return [tgt(img, 1000 + 20 * i, 1000, 1010 + 20 * i, 1010, cls) for i in range(k)]


def case(outs, targets, thr=0.5, expect=None):
    return {"outs": [rows(*o) if o else np.zeros((0, 6), f32) for o in outs], "targets": rows(*targets), "thr": thr,
            "expect": expect}


# (0,0,9,9) against (0,0,9,19): inter 100, union 200, IoU exactly 0.5 in fp32
HALF_P, HALF_T = (0, 0, 9, 9), (0, 0, 9, 19)


def iou_at_threshold(thr):
    tp = 1 if f32(0.5) >= f32(thr) else 0
    return case([[det(*HALF_P)]], [tgt(0, *HALF_T)], thr, [[tp]])


def tie_layout(i, j, first_is_left):
    """Image 0 holds two annotations at global target indices i < j (the other rows are image 1's).  The box P ties them
    (IoU 400/600 with both); LEFT and RIGHT are the two tied boxes.  Predictions: P, then RIGHT, then LEFT.
    The first maximum in target order wins: P claims the annotation at index i."""
    left, right = (10, 10, 29, 39), (10, 0, 29, 29)
    P = (10, 10, 29, 29)
    n = max(i, j) + 3
    t = filler(1, n)
    t[i] = tgt(0, *(left if first_is_left else right))
    t[j] = tgt(0, *(right if first_is_left else left))
    # P claims the box at index i; the exact copy of that box is then a claimed best (0), the other one is free (1)
    expect = [1, 1, 0] if first_is_left else [1, 0, 1]
    return case([[det(*P, conf=0.9), det(*right, conf=0.8), det(*left, conf=0.7)], []], t, 0.5, [expect, []])


def tie_first_claimed(i, j):
    """The first tied annotation is claimed before the tie: the tying prediction is a false positive although an equal
    annotation (the second) is unclaimed."""
    left, right = (10, 10, 29, 39), (10, 0, 29, 29)
    n = max(i, j) + 3
    t = filler(1, n)
    t[i], t[j] = tgt(0, *left), tgt(0, *right)
    return case([[det(*left, conf=0.9), det(10, 10, 29, 29, conf=0.8), det(*right, conf=0.7)], []], t, 0.5, [[1, 0, 1], []])


def claims_across_labels():
    """The best annotation has another label than the prediction: all annotations compete, so it is claimed anyway."""
    a, b = (0, 0, 19, 19), (0, 0, 19, 29)               # IoU(a, b) = 400 / 600
    t = [tgt(0, *b, cls=1), tgt(0, *a, cls=2)]
    outs = [[det(*a, cls=1, conf=0.9),                  # best is a (label 2), IoU 1: TP, claims a
             det(*a, cls=1, conf=0.8),                  # a again: claimed, FP
             det(*b, cls=2, conf=0.7)]]                 # label 2 exists; best is b (label 1), IoU 1: TP
    return case(outs, t, 0.5, [[1, 0, 1]])


def label_skip():
    """A prediction whose label no annotation of its image has is skipped and claims nothing."""
    a = (5, 5, 44, 44)
    t = [tgt(0, *a, cls=4), tgt(1, *a, cls=7)]           # label 7 exists in the batch, but not in image 0
    outs = [[det(*a, cls=7, conf=0.9), det(*a, cls=4, conf=0.8)], [det(*a, cls=4, conf=0.9), det(*a, cls=7, conf=0.8)]]
    return case(outs, t, 0.5, [[0, 1], [0, 1]])


def stop_rule():
    """Once every annotation is matched the loop stops: later perfect matches stay 0."""
    a, b = (0, 0, 9, 9), (50, 50, 69, 69)
    outs = [[det(*a, conf=0.9), det(*b, conf=0.8), det(*a, conf=0.7), det(*b, conf=0.6), det(0, 0, 9, 9, cls=1, conf=0.5)]]
    return case(outs, [tgt(0, *a), tgt(0, *b), tgt(1, *a, cls=1)], 0.5, [[1, 1, 0, 0, 0]])


def degenerate_boxes():
    """Zero-width boxes (x2 == x1: one pixel wide) and inverted ones (x2 < x1: negative area) on both sides."""
    t = [tgt(0, 10, 10, 10, 30), tgt(0, 40, 10, 30, 30), tgt(0, 60, 60, 80, 80), tgt(0, 100, 100, 99, 99)]
    outs = [[det(10, 10, 10, 30, conf=0.9), det(40, 10, 30, 30, conf=0.8), det(80, 60, 60, 80, conf=0.7),
             det(60, 60, 80, 80, conf=0.6), det(100, 100, 99, 99, conf=0.5), det(10, 10, 10, 30, conf=0.4)]]
    return case(outs, t, 0.5)


def nan_target():
    """A NaN coordinate makes that annotation's IoU NaN, and torch's max(0) returns it (the first NaN, before or after the
    largest number): no prediction of such an image is a true positive, although another annotation matches it exactly."""
    a = (0, 0, 19, 19)
    t = [tgt(0, NAN, 0, 19, 19), tgt(0, *a), tgt(1, *a), tgt(1, 0, NAN, 19, 19), tgt(1, 0, 0, 19, NAN)] + filler(2, 40)
    t += [tgt(2, *a), tgt(2, 0, 0, NAN, 19)]                # image 2: the NaN row a chunk after the match
    outs = [[det(*a, conf=0.9), det(*a, conf=0.8)], [det(*a)], [det(*a)]]
    return case(outs, t, 0.5, [[0, 0], [0], [0]])


def nan_inf_prediction():
    """A NaN coordinate in a prediction makes every IoU NaN (no TP, nothing claimed); an infinite one an empty overlap."""
    a, b = (0, 0, 19, 19), (30, 30, 49, 49)
    outs = [[det(NAN, 0, 19, 19, conf=0.9), det(*a, conf=0.8), det(30, 30, INF, 49, conf=0.7), det(30, 30, 49, NAN, conf=0.6),
             det(-INF, 30, 49, 49, conf=0.5), det(*b, conf=0.4)]]
    return case(outs, [tgt(0, *a), tgt(0, *b)], 0.5, [[0, 1, 0, 0, 0, 1]])


def empty_images():
    """Images without annotations, images without detections, and both."""
    outs, tg = synth.make_eval_case(401, 9, max_det=30, max_gt=6)
    tg = tg[np.isin(tg[:, 0], (0, 2, 3, 7))]            # images 1, 4, 5, 6, 8 keep no annotation
    for i in (3, 4, 8):
        outs[i] = np.zeros((0, 6), f32)                 # count 0
    return {"outs": outs, "targets": tg, "thr": 0.5, "expect": None}


def shuffled_targets(seed, n):
    """Targets of several images interleaved rather than grouped by image."""
    outs, tg = synth.make_eval_case(seed, n, max_det=60, max_gt=12, classes=5)
    rs = np.random.RandomState(seed + 1)
    return {"outs": outs, "targets": tg[rs.permutation(len(tg))], "thr": 0.5, "expect": None}


def random_degenerate(seed, n):
    """Seeded cases where a third of the boxes on both sides are inverted or zero-width."""
    outs, tg = synth.make_eval_case(seed, n, max_det=40, max_gt=9, classes=4)
    rs = np.random.RandomState(seed + 2)
    for a, c0 in [(o, 0) for o in outs] + [(tg, 2)]:     # column of x1 (x2 is two further)
        k = rs.rand(len(a)) < 0.33
        sw = rs.rand(len(a)) < 0.5
        lo, hi = a[:, c0].copy(), a[:, c0 + 2].copy()
        a[k & sw, c0], a[k & sw, c0 + 2] = hi[k & sw], lo[k & sw]          # inverted
        a[k & ~sw, c0 + 2] = a[k & ~sw, c0]                                 # zero width
    return {"outs": outs, "targets": tg, "thr": 0.5, "expect": None}


def large_batch(seed=402, n=4096, max_gt=10):
    """Many images, more annotations in total than fit a per-batch bitmask of 8192."""
    outs, tg = synth.make_eval_case(seed, n, max_det=24, max_gt=max_gt, classes=8)
    return {"outs": outs, "targets": tg, "thr": 0.5, "expect": None}


def crowded_image(n_ann=8500, n_det=300, seed=403):
    """One image with more than 8192 annotations (and a small second one)."""
    rs = np.random.RandomState(seed)
    c = rs.rand(n_ann, 2) * 2000
    wh = 4 + rs.rand(n_ann, 2) * 40
    t = np.zeros((n_ann, 6), f32)
    t[:, 1] = rs.randint(0, 3, n_ann)
    t[:, 2:4], t[:, 4:6] = c - wh / 2, c + wh / 2
    pick = rs.randint(0, n_ann, n_det)
    d = np.zeros((n_det, 6), f32)
    d[:, :4] = t[pick, 2:6] + rs.randn(n_det, 4).astype(f32) * np.where(rs.rand(n_det, 1) < 0.7, 1.0, 8.0).astype(f32)
    d[:, 5] = np.where(rs.rand(n_det) < 0.9, t[pick, 1], 3)
    d[:, 4] = np.sort(rs.rand(n_det).astype(f32))[::-1]
    d[rs.rand(n_det) < 0.1, :4] = d[0, :4]              # repeated boxes: claimed bests
    o2, t2 = synth.make_eval_case(seed + 1, 1, max_det=20, max_gt=5, classes=3)
    t2[:, 0] = 1
    return {"outs": [d, o2[0]], "targets": np.concatenate([t, t2]), "thr": 0.5, "expect": None}


THRESHOLDS = {"0.5": 0.5, "above": float(np.nextafter(f32(0.5), f32(1))), "below": float(np.nextafter(f32(0.5), f32(0))),
              "f64_rounds_to_half": 0.5 + 2.0 ** -30}

CASES = {
    **{"iou_at_threshold_" + k: (lambda v=v: iou_at_threshold(v)) for k, v in THRESHOLDS.items()},
    "tie_same_lane_left_first": lambda: tie_layout(3, 35, True),
    "tie_same_lane_right_first": lambda: tie_layout(3, 35, False),
    "tie_same_chunk_left_first": lambda: tie_layout(3, 17, True),
    "tie_same_chunk_right_first": lambda: tie_layout(17, 30, False),
    "tie_other_chunk_left_first": lambda: tie_layout(5, 40, True),
    "tie_other_chunk_right_first": lambda: tie_layout(30, 33, False),
    "tie_first_claimed_same_lane": lambda: tie_first_claimed(1, 65),
    "tie_first_claimed_other_chunk": lambda: tie_first_claimed(31, 32),
    "claims_across_labels": claims_across_labels,
    "label_skip": label_skip,
    "stop_rule": stop_rule,
    "degenerate_boxes": degenerate_boxes,
    "nan_target": nan_target,
    "nan_inf_prediction": nan_inf_prediction,
    "empty_images": empty_images,
    "shuffled_targets_5": lambda: shuffled_targets(404, 5),
    "n1": lambda: shuffled_targets(405, 1),
    "n5": lambda: random_degenerate(406, 5),
    "n7": lambda: shuffled_targets(407, 7),
}

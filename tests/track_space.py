"""Inputs of the tracker's space tests (test infrastructure), and the conditions each was built to reach.

yfv2_track_update's parallel code has work that small scenes never give it: augmenting paths of many steps over more than 128
solver columns (so one thread owns several columns, and the argmin combines lanes and warps), ties among columns of one thread,
of two lanes and of two warps, both orientations of the solver at scale, compactions of more than one 128-round, costs exactly
at a threshold, non-default parameters, capacities that are not a multiple of 4, 4096 streams in one call, extreme Kalman
states, and confidences near DBL_MAX, whose duals leave the finite numbers.  Each case below is a track_cases-style dict (S, K,
params, steps) with `claims`: (text, predicate) pairs on `reached(case)`, what tests/track_oracle.py's instrumentation says the
case reached.  An update step may carry a fourth element, the counts of the call (default: the number of rows of each stream).
Everything here is numpy; nothing needs a GPU."""
import math

import numpy as np

import track_cases as tc
import track_oracle as to

DBL_MAX = float(np.finfo(np.float64).max)


def box(x, y, w, h, conf, cls=0.0):
    return (x, y, x + w, y + h, conf, cls)


def arrays(step):
    d, n = tc.to_arrays(step[2])
    if len(step) > 3:
        n = np.asarray(step[3], np.int32)
    return d, n


def run_oracle(case, scalar=False):
    """Runs the case on the oracle with its instrumentation.  Returns (tracker, [(rows, counts, dropped) of each update])."""
    tr = to.Tracker(case["S"], case["K"], scalar=scalar, log=not scalar, **case["params"])
    outs = []
    for step in case["steps"]:
        if step[0] == "reset":
            tr.reset(step[1])
            continue
        d, n = arrays(step)
        outs.append(tr.update(d, n, step[1]))
    return tr, outs


def reached(case):
    """What the oracle's instrumentation saw on the case: path steps (sweeps of the argmin) and augmenting path lengths, in all
    stages and in stages of more than 128 columns, the owner kinds of the argmin's ties, the orientations, the sizes of the
    reduced problems, the duplicate rule's pairs and whether a dual left the finite numbers."""
    tr, outs = run_oracle(case)
    st = [g for g in tr.log if g["stage"] != "dup" and "steps" in g]
    wide = [g for g in st if g["ncol"] > 128]
    r = dict(
        stages=len(st),
        max_steps=max([max(g["steps"]) for g in st] or [0]),
        max_path=max([max(g["plen"]) for g in st] or [0]),
        max_steps_wide=max([max(g["steps"]) for g in wide] or [0]),
        steps_wide=sum(sum(g["steps"]) for g in wide),
        max_cols=max([g["ncol"] for g in st] or [0]),
        ties=set().union(*[g["ties"] for g in st]) if st else set(),
        tr={g["tr"] for g in st},
        ties_by_tr={o: set().union(*[g["ties"] for g in st if g["tr"] == o]) for o in (False, True)},
        rounds=max([max(-(-g["nt"] // to.NT), -(-g["nd"] // to.NT)) for g in tr.log if "nt" in g] or [0]),
        reduced_both=any(g["ntr"] < g["nt"] and g["ndr"] < g["nd"] and g["nt"] > to.NT and g["nd"] > to.NT for g in st),
        dup_pairs=max([g["pairs"] for g in tr.log if g["stage"] == "dup"] or [0]),
        nonfinite=any(g["nonfinite"] for g in st),
        dropped=sum(sum(o[2]) for o in outs),
        tracker=tr, outs=outs)
    return r


# ---- crowds --------------------------------------------------------------------------------------------------------------------
def crowd(seed, n=600, frames=6, K=1024, spacing=16.0, side=24.0, huge=False):
    """n objects on a jittered grid, spaced closer than their width, drifting; each frame drops some (lost tracks, found again
    later), reports some at low confidence (stage 2), adds new ones (tentative tracks: stage 3 on the next frame) and clutter.
    huge: a third of the high confidences are 1e300 .. DBL_MAX."""
    rng = np.random.default_rng(seed)
    g = int(math.ceil(math.sqrt(n)))
    p = np.stack([np.arange(n) % g, np.arange(n) // g], 1) * spacing + rng.uniform(-4, 4, (n, 2)) + 50
    v = rng.normal(0, 1.5, (n, 2))
    born = np.zeros(n, bool)
    born[rng.permutation(n)[:int(0.8 * n)]] = True
    steps = []
    for f in range(frames):
        p = p + v
        if f:
            born |= rng.random(n) < 0.1
        rows = []
        for k in np.flatnonzero(born):
            if rng.random() < 0.12:
                continue
            c = p[k] + rng.normal(0, 1.0, 2)
            wh = side * (1 + rng.normal(0, 0.05, 2))
            conf = float(rng.uniform(0.15, 0.45)) if rng.random() < 0.2 else float(rng.uniform(0.55, 1.0))
            if huge and conf > 0.5 and rng.random() < 0.35:
                conf = float(rng.choice([1e300, 1e306, 1e307, 8e307, 1.7e308, DBL_MAX]))
            rows.append(tc.det(float(c[0]), float(c[1]), float(wh[0]), float(wh[1]), conf))
        for _ in range(int(rng.integers(0, 6))):
            rows.append(tc.det(*rng.uniform([50, 50, 10, 10], [50 + g * spacing, 50 + g * spacing, 40, 40]).tolist(),
                               float(rng.uniform(0.05, 0.9))))
        steps.append(("update", [0], [[rows[i] for i in rng.permutation(len(rows))]]))
    return dict(name="crowd_%d_%d%s" % (n, seed, "_huge" if huge else ""), S=1, K=K, params=dict(max_age=3), steps=steps)


# ---- staircase: the new row displaces every earlier one ------------------------------------------------------------------------
def staircase(n=300, dets_as_rows=False):
    """n + 1 boxes (the solver's columns) at x = 8j, width 12, and n boxes (its rows, in this order) between them: row r < n - 1
    between columns n-1-r and n-r, 0.002 px to the left, so it takes its left column; the last row sits 1 px from column 1.
    Every earlier row then moves one column to the right: one augmenting path through all n rows.  dets_as_rows: the columns
    are the tracks and the rows the detections (the solver's swapped orientation), else the other way round."""
    cols = [box(8.0 * j - 6, 100.0, 12.0, 12.0, 1.0) for j in range(n + 1)]
    xs = [8.0 * (n - r - 0.5) - 0.002 for r in range(n - 1)] + [7.0]
    rows = [box(x - 6, 100.0, 12.0, 12.0, 1.0) for x in xs]
    first, second = (cols, rows) if dets_as_rows else (rows, cols)
    first = [r[:4] + (0.9, 0.0) for r in first]
    return dict(name="staircase_%d_%s" % (n, "dets_as_rows" if dets_as_rows else "tracks_as_rows"), S=1, K=512, params={},
                steps=[("update", [0], [first]), ("update", [0], [second])])


# ---- ties across column owners -------------------------------------------------------------------------------------------------
TIE_OFFSETS = (0, 1, 32, 128, 129, 160)


def ties(dets_as_rows=False, base=3, ncol=200):
    """Identical boxes at reduced columns base + (0, 1, 32, 128, 129, 160): one thread's two columns, two lanes, two warps.  The
    other columns are fillers, each with its own partner far away.  Two identical partners on the tied spot make the second
    path run through the first and meet the tie again.  dets_as_rows: the tied columns are tracks (ids in that order) and the
    partners detections."""
    tied = {base + o for o in TIE_OFFSETS}
    spot = box(200.0, 200.0, 64.0, 64.0, 0.75)
    col, partners = [], [spot, spot]
    for j in range(ncol):
        if j in tied:
            col.append(spot)
        else:
            x, y = 1000.0 + 80.0 * (j % 20), 100.0 + 80.0 * (j // 20)
            col.append(box(x, y, 40.0, 40.0, 0.9))
            partners.append(box(x + 2, y + 1, 40.0, 40.0, 0.9))
    tracks, dets = (col, partners) if dets_as_rows else (partners, col)
    tracks = [r[:4] + (0.9, 0.0) for r in tracks]
    return dict(name="ties_%s" % ("dets_as_rows" if dets_as_rows else "tracks_as_rows"), S=1, K=256, params={},
                steps=[("update", [0], [tracks]), ("update", [0], [dets]), ("update", [0], [dets])])


# ---- sparse reductions ---------------------------------------------------------------------------------------------------------
def sparse(seed=0, nt=640, nd=1600, paired=300):
    """nt tracks on a grid, then nd detections of which only `paired` overlap a track (some two at once); the rest are far."""
    rng = np.random.default_rng(seed)
    g = 32
    tp = [(60.0 + 50 * (k % g), 60.0 + 50 * (k // g)) for k in range(nt)]
    f1 = [tc.det(x, y, 30, 30, 0.9) for x, y in tp]
    f2 = []
    for k in rng.choice(nt, paired, replace=False):
        x, y = tp[k]
        f2.append(tc.det(x + float(rng.normal(0, 2)), y + float(rng.normal(0, 2)), 30, 30, float(rng.uniform(0.55, 1.0))))
    while len(f2) < nd:
        f2.append(tc.det(*rng.uniform([3000, 0, 10, 10], [6000, 3000, 40, 40]).tolist(), float(rng.uniform(0.55, 1.0))))
    f2 = [f2[i] for i in rng.permutation(nd)]
    return dict(name="sparse", S=1, K=1024, params={}, steps=[("update", [0], [f1]), ("update", [0], [f2])])


# ---- at the limits, with contention ----------------------------------------------------------------------------------------------
def limits_contended(seed=0, K=1024, M=2048, frames=3):
    """K tracks on a grid of spacing 16 with boxes of 24, then frames of M rows: two jittered rows on each track, three in four
    high, so each track overlaps 2-4 high detections (its own and its neighbours') and some low ones."""
    rng = np.random.default_rng(seed)
    g = int(math.ceil(math.sqrt(K)))
    p = np.stack([np.arange(K) % g, np.arange(K) // g], 1) * 16.0 + 40
    steps = [("update", [0], [[tc.det(float(x), float(y), 24, 24, 0.9) for x, y in p]])]
    for f in range(frames - 1):
        rows = []
        for k in range(M):
            x, y = p[k % K] + rng.uniform(-5, 5, 2)
            conf = float(rng.uniform(0.55, 1.0)) if rng.random() < 0.75 else float(rng.uniform(0.15, 0.45))
            rows.append(tc.det(float(x), float(y), float(rng.uniform(20, 28)), float(rng.uniform(20, 28)), conf))
        steps.append(("update", [0], [[rows[i] for i in rng.permutation(M)]]))
    return dict(name="limits_contended", S=1, K=K, params={}, steps=steps)


# ---- exact thresholds ------------------------------------------------------------------------------------------------------------
def walk(f, x, target, up):
    """The float x', reached from x by single-ulp steps, with f(x') == target; f is monotone, increasing in x when up."""
    for _ in range(1 << 16):
        y = f(x)
        if y == target:
            return x
        x = float(np.nextafter(x, math.inf if (y < target) == up else -math.inf))
    raise AssertionError("walk: no float reaches %r" % target)


def track_box(row):
    """The box of a track born on `row` (zero velocity: predicting does not move it)."""
    return to.box(list(to.measure(row[:4])))


def cost(track_row, det_row, fused):
    q = to.iou(track_box(track_row), det_row[:4])
    return 1.0 - (q * det_row[4] if fused else q)


def targets(thr):
    """The cost exactly at thr and the nearest costs on either side that 1 - x can give (none above 1: it would need a negative
    IoU; below 0.5 the nearest is 0.5 - 2^-53, as 1 - x has no finer step there)."""
    below = 0.5 - 2.0 ** -53 if thr == 0.5 else float(np.nextafter(thr, 0.0))
    out = [(below, True), (thr, False)]
    return out + ([(float(np.nextafter(thr, 2.0)), False)] if thr < 1.0 else [])


def fused_cell(origin, c, q):
    """A track row and a detection row (IoU about q, confidence walked) whose fused cost is exactly c."""
    x0, y0 = origin
    t = box(x0, y0, 64.0, 64.0, 0.9)
    if q < 1e-10:
        e = 2.0 ** -47 if c == 1.0 else 2.0 ** -46                   # a sliver: IoU 2^-54 or 2^-53
        d = box(x0 + 64.0 - e, y0, 64.0, 64.0, 0.0)
    else:
        dx = round(64.0 * (1 - q) / (1 + q) * 1024) / 1024
        d = box(x0 + dx, y0, 64.0, 64.0, 0.0)
    q = to.iou(track_box(t), d[:4])
    conf = walk(lambda k: 1.0 - q * k, min(1.0, max(0.75, (1.0 - c) / q)), c, False)
    return t, d[:4] + (conf, 0.0)


def thresholds_stage1(match_thresh):
    """Stage 1 (fused, thr = match_thresh): one confirmed track per cell, one high detection per cell at a cost one ulp below,
    at, or one ulp above the threshold."""
    cells = []
    for k, (c, allowed) in enumerate(targets(match_thresh)):
        t, d = fused_cell((0.0, 128.0 * k), c, (1.0 - match_thresh) / 0.8)
        cells.append(dict(track=t, det=d, cost=c, allowed=allowed, fused=True))
    steps = [("update", [0], [[x["track"] for x in cells]]), ("update", [0], [[x["det"] for x in cells]])]
    return dict(name="thr_stage1_%g" % match_thresh, S=1, K=8, params=dict(match_thresh=match_thresh), steps=steps, cells=cells,
                thr=match_thresh)


def thresholds_stage2():
    """Stage 2 (1 - IoU, thr 0.5): a confirmed track without a high detection, and one low detection over it whose height is
    walked so that 1 - IoU is 0.5 or the nearest cost on either side that 1 - IoU can reach (0.5 -+ 2^-53)."""
    cells = []
    for k, (c, allowed) in enumerate([(0.5 - 2.0 ** -53, True), (0.5, False), (0.5 + 2.0 ** -53, False)]):
        x0 = 1024.0 * k
        t = box(x0, 0.0, 64.0, 64.0, 0.9)
        h = walk(lambda hh: cost(t, (x0, 0.0, x0 + 64.0, hh, 0.3), False), 128.0, c, True)
        cells.append(dict(track=t, det=(x0, 0.0, x0 + 64.0, h, 0.3, 0.0), cost=c, allowed=allowed, fused=False))
    steps = [("update", [0], [[x["track"] for x in cells]]), ("update", [0], [[x["det"] for x in cells]])]
    return dict(name="thr_stage2", S=1, K=8, params={}, steps=steps, cells=cells, thr=to.STAGE2_THR)


def thresholds_stage3():
    """Stage 3 (fused, thr 0.7): tentative tracks (born on frame 2) and high detections on frame 3 around 0.7."""
    cells = []
    for k, (c, allowed) in enumerate(targets(to.STAGE3_THR)):
        t, d = fused_cell((0.0, 128.0 * k), c, 0.3 / 0.8)
        cells.append(dict(track=t, det=d, cost=c, allowed=allowed, fused=True))
    far = [box(5000.0, 5000.0, 16.0, 16.0, 0.9)]
    steps = [("update", [0], [far]), ("update", [0], [[x["track"] for x in cells]]), ("update", [0], [[x["det"] for x in cells]])]
    return dict(name="thr_stage3", S=1, K=8, params={}, steps=steps, cells=cells, thr=to.STAGE3_THR)


def duplicate_rule():
    """The duplicate rule at IoU exactly 0.85 and one ulp above, with equal ages (frame-1 twins, the detection stays on one: the
    tracked one goes) and unequal ones (a twin born on frame 2 and lost on frame 4: the older tracked one stays).  Every
    detection sits exactly on its track, so updates leave the means, and so the boxes, as they were born."""
    streams, pairs = [], []
    for target, ah in ((to.DUP_IOU, 102.0), (float(np.nextafter(to.DUP_IOU, 1.0)), 64.0)):
        a = box(0.0, 0.0, 64.0, ah, 1.0)                            # b: a taller box over a, its height walked
        bh = walk(lambda h: to.iou(track_box(a), track_box(box(0.0, 0.0, 64.0, h, 0.9))), ah / 0.85, target, False)
        b = box(0.0, 0.0, 64.0, bh, 1.0)
        pairs.append(target)
        streams.append([[a, b], [b], [b], [b]])                    # equal ages
        streams.append([[a], [a, b], [a, b], [a]])                 # A older, B lost on frame 4
    steps = [("update", list(range(len(streams))), [s[f] for s in streams]) for f in range(4)]
    return dict(name="dup_rule", S=len(streams), K=8, params=dict(match_thresh=0.05), steps=steps, ious=pairs)


# ---- where the reduction's edges change the matching ---------------------------------------------------------------------------
def reduction_edges():
    """Two small scenes on a 16 px lattice under match_thresh 0.5 and confidence 1 (stage-1 cost 1 - IoU, exact), found by a
    search over lattice boxes: in stream 0 a track and a detection whose only pair sits exactly at the threshold would, if let
    into the reduced problem, flip the solver's orientation and with it the tie among equal optima; in stream 1 the reduced
    problem is square, so the tracks are the rows (swapping sides on equal sizes picks the other optimum)."""
    scenes = [([(1, 2, 2, 5), (1, 2, 2, 5), (0, 2, 2, 3), (0, 0, 1, 3)], [(0, 1, 2, 3), (3, 0, 5, 1), (1, 2, 2, 4), (3, 3, 4, 5)]),
              ([(1, 1, 4, 4), (1, 1, 4, 4), (2, 1, 5, 3)], [(0, 0, 1, 1), (1, 1, 4, 4), (2, 0, 5, 3), (3, 1, 5, 3)])]
    rows = [[tuple(16.0 * v for v in b) + (c, 0.0) for b in bs] for scene in scenes for bs, c in zip(scene, (0.9, 1.0))]
    return dict(name="reduction_edges", S=2, K=8, params=dict(match_thresh=0.5),
                steps=[("update", [0, 1], [rows[0], rows[2]]), ("update", [0, 1], [rows[1], rows[3]])], scenes=scenes)


# ---- non-default parameters ------------------------------------------------------------------------------------------------------
PARAMS = {
    "low0": dict(low_thresh=0.0),
    "high_eq_new": dict(high_thresh=0.6, new_thresh=0.6),
    "new1": dict(new_thresh=1.0),
    "age0": dict(max_age=0),
    "match1": dict(match_thresh=1.0),
    "match005": dict(match_thresh=0.05),
}


def with_params(name, seed=4):
    """A seeded 6-stream scene under non-default parameters; confidences above 0.9 become exactly 1 (births under new_thresh 1),
    and each frame of stream 0 adds rows at confidence 0 and 5e-324 (used only under low_thresh 0)."""
    c = tc.scene(seed, S=6, frames=16, K=32, max_objects=10)
    steps = []
    for st in c["steps"]:
        if st[0] == "update":
            rows_all = [[r[:4] + (1.0 if r[4] > 0.9 else r[4], r[5]) for r in rows] for rows in st[2]]
            if 0 in st[1]:
                rows_all[st[1].index(0)] += [tc.det(900, 500, 40, 40, 0.0), tc.det(300, 700, 40, 40, 5e-324)]
            st = ("update", st[1], rows_all)
        steps.append(st)
    return dict(name="params_" + name, S=c["S"], K=c["K"], params=dict(c["params"], **PARAMS[name]), steps=steps)


# ---- capacity ----------------------------------------------------------------------------------------------------------------------
def capacity(K, seed=0, S=3, frames=4):
    """Capacity K (not a multiple of 4 except through the rounding of the layout): S streams with K + 1 .. K + 40 distinct objects,
    some missing on each frame, so births are refused (counted in dropped, spending no id) while lost tracks hold slots."""
    rng = np.random.default_rng(seed)
    steps, objs = [], []
    for s in range(S):
        n = K + int(rng.integers(1, 41))
        objs.append([(40.0 + 40 * (k % 40) + 5000 * s, 40.0 + 40 * (k // 40)) for k in range(n)])
    for f in range(frames):
        streams = [int(s) for s in rng.permutation(S)]
        rows_all = []
        for s in streams:
            rows = [tc.det(x + f, y, 24, 24, float(rng.uniform(0.6, 1.0))) for x, y in objs[s] if rng.random() > 0.1 * f]
            rows_all.append([rows[i] for i in rng.permutation(len(rows))])
        steps.append(("update", streams, rows_all))
    return dict(name="capacity_%d" % K, S=S, K=K, params=dict(max_age=1), steps=steps)


# ---- many streams --------------------------------------------------------------------------------------------------------------------
def many_streams(seed=0, S=5000, B=4096, K=3, M=6, frames=3):
    """B = 4096 of S = 5000 streams per call (the launch's limit), in shuffled order, capacity 3: most streams empty or with one to
    six objects; some calls give a stream counts above M (read as M) or negative (read as 0).  The same S - B streams sit out every
    call, so their state must not change."""
    rng = np.random.default_rng(seed)
    called = [int(s) for s in rng.permutation(S)[:B]]
    objs = {s: [rng.uniform([50, 50], [1800, 1000]) for _ in range(int(rng.integers(0, M + 1)) if rng.random() < 0.6 else 0)]
            for s in called}
    steps = []
    for f in range(frames):
        streams = [called[i] for i in rng.permutation(B)]
        rows_all, counts = [], []
        for s in streams:
            rows = [tc.det(float(p[0]) + 3 * f, float(p[1]), 60, 90, float(rng.uniform(0.55, 1.0))) for p in objs[s]]
            rows_all.append(rows)
            u = rng.random()
            counts.append(M + 5 if u < 0.03 else (-3 if u < 0.06 else len(rows)))
        steps.append(("update", streams, rows_all, counts))
    return dict(name="many_streams", S=S, K=K, params={}, steps=steps, called=called)


# ---- Kalman extremes -----------------------------------------------------------------------------------------------------------------
def kalman_extremes(frames=8):
    """Streams of one object each: sides of 1e-3 px and 1e6 px, aspect ratios 1e-4 and 1e4, and two whose aspect flips between 0.2
    and 5 every frame (one beside a steady twin).  The flip does not drive the predicted aspect negative: its velocity noise
    (1e-5) keeps the aspect's gain for velocity near 0, so the flipping object loses its track and starts new ones instead."""
    rng = np.random.default_rng(0)
    shapes = [(1e-3, 1e-3), (1e6, 1e6), (1e-2, 1e2), (1e4, 1.0)]
    streams = []
    for w, h in shapes:
        streams.append([[tc.det(5.0 * f + w * 0.01 * float(rng.normal()), 3.0 * f, w * (1 + 0.01 * float(rng.normal())), h, 0.9)]
                        for f in range(frames)])
    streams.append([[tc.det(500.0 + f, 500.0, 40.0 if f % 2 else 200.0, 200.0 if f % 2 else 40.0, 0.9)] for f in range(frames)])
    streams.append([[tc.det(500.0, 500.0, 40.0 * (1 + 4 * (f % 2)), 200.0, 0.9), tc.det(520.0, 500.0, 40.0, 200.0, 0.9)]
                    for f in range(frames)])
    steps = [("update", list(range(len(streams))), [s[f] for s in streams]) for f in range(frames)]
    return dict(name="kalman_extremes", S=len(streams), K=8, params=dict(max_age=2), steps=steps)


# ---- the cases and their claims --------------------------------------------------------------------------------------------------------
def exact_pair(scene, thr):
    return bool((1.0 - to.iou_matrix(np.array(scene[0], np.float64), np.array(scene[1], np.float64)) == thr).any())


def cases():
    out = []

    def add(case, *claims):
        case["claims"] = list(claims)
        out.append(case)

    add(crowd(1), ("a path of >= 20 steps over > 128 columns", lambda r: r["max_steps_wide"] >= 20),
        ("all three stages ran", lambda r: {g["stage"] for g in r["tracker"].log} >= {1, 2, 3}))
    add(crowd(2, n=1000, frames=4), ("a path of >= 20 steps over > 128 columns", lambda r: r["max_steps_wide"] >= 20))
    for rows_dets in (False, True):
        add(staircase(300, rows_dets), ("an augmenting path through >= n/2 rows", lambda r: r["max_path"] >= 150),
            ("orientation", lambda r, o=rows_dets: o in r["tr"]))
        add(ties(rows_dets), ("ties of one thread, two lanes and two warps", lambda r, o=rows_dets: r["ties_by_tr"][o] >= {"thread", "lane", "warp"}),
            ("more than 128 columns", lambda r: r["max_cols"] > 128))
    add(sparse(), ("compactions of more than one round", lambda r: r["rounds"] > 1),
        ("the reduced problem smaller on both sides", lambda r: r["reduced_both"]))
    add(limits_contended(), ("a path of >= 20 steps over > 128 columns", lambda r: r["max_steps_wide"] >= 20),
        ("births refused at capacity", lambda r: r["dropped"] > 0))
    for m in (0.8, 0.5, 1.0):
        add(thresholds_stage1(m))
    add(thresholds_stage2())
    add(thresholds_stage3())
    add(duplicate_rule())
    add(reduction_edges(), ("stream 0 has a pair exactly at the threshold", lambda r: exact_pair(reduction_edges()["scenes"][0], 0.5)),
        ("stream 1 solves a square problem", lambda r: any(g["stream"] == 1 and g["stage"] == 1 and g["ntr"] == g["ndr"]
                                                            for g in r["tracker"].log if "ntr" in g)))
    for name in PARAMS:
        add(with_params(name))
    for K in (1, 3, 5, 127, 129, 1023):
        add(capacity(K), ("births refused", lambda r: r["dropped"] > 0))
    add(kalman_extremes(), ("flips refused matches: births after frame 1", lambda r: r["tracker"].streams[4]["next_id"] > 2))
    add(crowd(3, n=300, frames=5, huge=True), ("a dual left the finite numbers", lambda r: r["nonfinite"]))
    return out


def by_name():
    return {c["name"]: c for c in cases()}

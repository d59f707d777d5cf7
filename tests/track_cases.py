"""Inputs of the tracker tests (test infrastructure): hand-built sequences for each rule of the lifecycle, seeded scenes of moving
objects, and the dense and limit frames.  A case is a dict: S streams, capacity K, tracker params, and steps, each ("update",
streams, [rows of each stream]) or ("reset", streams); rows are (x1, y1, x2, y2, conf, cls) in frame pixels."""
import math

import numpy as np


def det(cx, cy, w, h, conf, cls=0.0):
    return (cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2, conf, cls)


def single(name, frames, K=16, **params):
    """One stream; frames: the rows of each frame."""
    return dict(name=name, S=1, K=K, params=params, steps=[("update", [0], [rows]) for rows in frames])


def hand_cases():
    A = det(100, 100, 40, 80, 0.9, 1.0)
    A2 = det(103, 101, 40, 80, 0.9, 1.0)
    far = det(400, 300, 30, 30, 0.9, 2.0)
    twin = det(101, 100, 40, 80, 0.8, 3.0)
    cases = [
        single("first_frame_confirmed", [[A, far], [A2, far]]),
        single("tentative_confirmed_on_second_frame", [[], [A], [A2], [A2]]),
        single("tentative_dropped_when_unmatched", [[], [A], [], [A]]),
        single("byte_low_score_keeps_track", [[A]] + [[det(100 + 2 * k, 100, 40, 80, 0.3, 5.0)] for k in range(1, 6)]),
        single("low_score_alone_starts_nothing", [[det(100, 100, 40, 80, 0.4)], [det(100, 100, 40, 80, 0.4)]]),
        single("lost_refound_keeps_id", [[A, far], [far], [far], [far], [A2, far]]),
        single("removed_at_max_age_plus_one", [[A]] + [[]] * 3 + [[A]], max_age=2),
        single("kept_at_max_age", [[A]] + [[]] * 2 + [[A]], max_age=2),
        # two frame-1 tracks on one object: the single detection of frame 2 goes to one, the other is lost, equal ages remove the
        # tracked one
        single("duplicate_equal_ages", [[A, twin], [A2]]),
        # a younger track (born frame 2 on a twin detection) next to an older one; frame 4's single detection sits on the older
        # (the lost younger one goes) or on the younger (the younger tracked one goes)
        single("duplicate_older_tracked", [[A], [A, twin], [A, twin], [A]]),
        single("duplicate_younger_tracked", [[A], [A, twin], [A, twin], [twin]]),
        single("births_past_capacity", [[A, far, det(250, 50, 20, 20, 0.95)], [A2, far, det(250, 50, 20, 20, 0.95), det(30, 30, 10, 10, 0.9)]],
               K=2),
        single("conf_at_each_threshold", [[det(50, 50, 20, 20, 0.1), det(150, 50, 20, 20, 0.5), det(250, 50, 20, 20, 0.6),
                                           det(350, 50, 20, 20, float(np.nextafter(0.6, 0.0))), det(450, 50, 20, 20, 1.0)]] * 2),
        single("invalid_rows", [[(10.0, 10.0, 10.0, 50.0, 0.9, 0.0), (10.0, 10.0, 50.0, 10.0, 0.9, 0.0), (60.0, 10.0, 50.0, 40.0, 0.9, 0.0),
                                 (math.nan, 10.0, 50.0, 50.0, 0.9, 0.0), (10.0, 10.0, math.inf, 50.0, 0.9, 0.0),
                                 (10.0, 10.0, 50.0, 50.0, math.nan, 0.0), (10.0, 10.0, 50.0, 50.0, 0.9, math.inf),
                                 (-math.inf, 10.0, 50.0, 50.0, 0.9, 0.0), A]]),
        single("crossing", [[det(100 + 20 * k, 100, 40, 80, 0.9, 0.0), det(300 - 20 * k, 104, 40, 80, 0.85, 1.0)] for k in range(12)]),
        dict(name="reset_restarts_ids_and_frames", S=2, K=8, params={},
             steps=[("update", [0, 1], [[A], [far]]), ("update", [1, 0], [[far], [A2, far]]), ("reset", [0]),
                    ("update", [0, 1], [[far], [far]]), ("update", [0], [[far]])]),
    ]
    return cases


def scene(seed, S=16, frames=40, K=64, max_objects=12, max_age=8, reset_at=None):
    """Seeded scenes of S streams: objects in linear motion with noise, some crossing, occlusion gaps shorter and longer than
    max_age, frames of low-score detections only, flicker of confidence and drop-outs, streams missing from calls, and a reset
    of some streams at frame `reset_at`."""
    rng = np.random.default_rng(seed)
    objs = []
    for s in range(S):
        n = int(rng.integers(1, max_objects + 1))
        o = []
        for _ in range(n):
            o.append(dict(p=rng.uniform([50, 50], [1800, 1000]), v=rng.normal(0, 6, 2), wh=rng.uniform([20, 40], [120, 240]),
                          cls=float(rng.integers(0, 5)), gap=(int(rng.integers(0, frames)), int(rng.choice([2, 3, max_age + 4])))))
        objs.append(o)
    steps, calls = [], [0] * S
    for f in range(frames):
        if reset_at is not None and f == reset_at:
            steps.append(("reset", sorted(rng.choice(S, size=max(1, S // 3), replace=False).tolist())))
        streams = [s for s in range(S) if rng.random() > 0.15]
        if not streams:
            streams = [0]
        rng.shuffle(streams)
        rows_all = []
        only_low = rng.random() < 0.1
        for s in streams:
            rows = []
            for o in objs[s]:
                o["p"] = o["p"] + o["v"]
                g0, gl = o["gap"]
                if g0 <= calls[s] < g0 + gl or rng.random() < 0.05:
                    continue
                wh = o["wh"] * (1 + rng.normal(0, 0.03, 2))
                c = o["p"] + rng.normal(0, 2.0, 2)
                conf = float(rng.uniform(0.15, 0.45)) if only_low or rng.random() < 0.15 else float(rng.uniform(0.5, 0.99))
                rows.append(det(float(c[0]), float(c[1]), float(wh[0]), float(wh[1]), conf, o["cls"]))
            for _ in range(int(rng.integers(0, 3))):                       # clutter
                rows.append(det(*rng.uniform([0, 0, 10, 10], [1920, 1080, 60, 60]).tolist(), float(rng.uniform(0.05, 0.7))))
            order = rng.permutation(len(rows))
            rows_all.append([rows[i] for i in order])
            calls[s] += 1
        steps.append(("update", streams, rows_all))
    return dict(name="scene_%d" % seed, S=S, K=K, params=dict(max_age=max_age), steps=steps)


def dense_ties(n=64):
    """n tracks on n objects stacked on one spot (confirmed on frame 1), then n detections that all overlap every track with
    equal costs in blocks: long augmenting paths and many ties."""
    f1 = [det(500 + (k % 8), 400 + (k // 8), 100, 200, 0.9) for k in range(n)]
    f2 = [det(500 + (k % 4), 400 + (k % 3), 100, 200, 0.6 + 0.3 * ((k * 7) % 5) / 4) for k in range(n)]
    return dict(name="dense_ties_%d" % n, S=1, K=n, params={}, steps=[("update", [0], [f1]), ("update", [0], [f2]),
                                                                       ("update", [0], [f1])])


def limits(K=1024, M=2048):
    """A frame at the limits: K tracks on a grid, then M rows per frame, the first K on the tracks and the rest far apart."""
    grid = int(math.ceil(math.sqrt(K)))
    f1 = [det(20 + 30 * (k % grid), 20 + 30 * (k // grid), 20, 20, 0.9) for k in range(K)]
    extra = [det(2000 + 30 * (k % 64), 20 + 30 * (k // 64), 20, 20, 0.3 if k % 2 else 0.9) for k in range(M - K)]
    f2 = [det(21 + 30 * (k % grid), 20 + 30 * (k // grid), 20, 20, 0.9 if k % 3 else 0.3) for k in range(K)] + extra
    return dict(name="limits", S=1, K=K, params={}, steps=[("update", [0], [f1]), ("update", [0], [f2])])


def to_arrays(rows_all):
    """The rows of each stream of a call -> (dets float64 [B, M, 6], counts int32 [B]), M >= 1."""
    M = max([1] + [len(r) for r in rows_all])
    dets = np.zeros((len(rows_all), M, 6), np.float64)
    for b, rows in enumerate(rows_all):
        if rows:
            dets[b, :len(rows)] = np.asarray(rows, np.float64)
    return dets, np.array([len(r) for r in rows_all], np.int32)

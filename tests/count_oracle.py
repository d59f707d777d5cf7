"""Restatement (test infrastructure) of the line and zone counter of yfv2_count_update (include/yfv2.h), driven by the outputs and
live set of tests/track_oracle.Tracker.  Records are keyed by track id, as the contract states them (the device keys them by
slot).  Every fp64 value is a Python float and every operation one IEEE fp64 operation with one rounding; the zone test is
cv2.pointPolygonTest(contour_f32, point_f32, False) >= 0 restated with numpy float32 differences and fp64 products, pinned to
cv2 by tests/golden/count_cases.npz."""
import numpy as np

import track_oracle as to

LINE, ENTRY, EXIT = 0, 1, 2


def orient(ax, ay, bx, by, px, py):
    return (bx - ax) * (py - ay) - (by - ay) * (px - ax)


def sign(v):
    return (v > 0.0) - (v < 0.0)


def anchor(box):
    """Bottom centre of a track's (x1, y1, x2, y2)."""
    return ((box[0] + box[2]) / 2, box[3])


def point_polygon(contour, x, y):
    """cv2.pointPolygonTest(contour, (x, y), False) of a float32 contour [n, 2] at a point already in float32: 1 inside, 0 on the
    boundary, -1 outside."""
    v = np.asarray(contour, np.float32)
    x, y = np.float32(x), np.float32(y)
    b = v
    a = np.roll(v, 1, axis=0)                       # a = the previous vertex of each edge, v[n-1] for the first
    skip = ((a[:, 1] <= y) & (b[:, 1] <= y)) | ((a[:, 1] > y) & (b[:, 1] > y)) | ((a[:, 0] < x) & (b[:, 0] < x))
    on = skip & (y == b[:, 1]) & ((x == b[:, 0]) | ((y == a[:, 1]) & (((a[:, 0] <= x) & (x <= b[:, 0])) | ((b[:, 0] <= x) & (x <= a[:, 0])))))
    with np.errstate(over="ignore", invalid="ignore"):
        dist = ((y - a[:, 1]).astype(np.float64) * (b[:, 0] - a[:, 0]).astype(np.float64)
                - (x - a[:, 0]).astype(np.float64) * (b[:, 1] - a[:, 1]).astype(np.float64))
    dist = np.where(b[:, 1] < a[:, 1], -dist, dist)
    if on.any() or (~skip & (dist == 0)).any():
        return 0
    return 1 if int((~skip & (dist > 0)).sum()) % 2 else -1


def inside(contour, q):
    """The contract's inside(Q): the fp64 anchor rounded to float32, the boundary inside."""
    return point_polygon(contour, np.float32(q[0]), np.float32(q[1])) >= 0


class Counter:
    """The counter state of S streams: geometry, records by id and totals."""

    def __init__(self, S):
        self.S = S
        self.geom = [([], []) for _ in range(S)]
        self.rec = [dict() for _ in range(S)]
        self.tot = [None] * S
        for s in range(S):
            self.set_geometry(s, [], [])

    def set_geometry(self, s, lines, zones):
        """lines: [(ax, ay, bx, by)], zones: [contour [n, 2]] (rounded to float32, as the device stores them)."""
        self.geom[s] = ([tuple(float(c) for c in g) for g in lines], [np.asarray(z).astype(np.float32) for z in zones])
        self.reset([s])

    def reset(self, streams):
        for s in streams:
            lines, zones = self.geom[s]
            self.rec[s] = {}
            self.tot[s] = {"lines": np.zeros((len(lines), 2), np.int64), "zones": np.zeros((len(zones), 2), np.int64)}

    def update(self, tracker, streams):
        """tracker: a track_oracle.Tracker after its update.  Returns (events: B lists of 8-tuples, counts [B], occupancy: B lists
        of the stream's zone counts)."""
        events, occupancy = [], []
        for s in streams:
            st = tracker.streams[s]
            lines, zones = self.geom[s]
            rec, tot = self.rec[s], self.tot[s]
            live = {t["id"] for t in st["tracks"]}
            for i in [i for i in rec if i not in live]:
                del rec[i]
            ev, occ = [], [0] * len(zones)
            for t in st["tracks"]:                                   # ascending id
                if not (t["state"] == to.TRACKED and t["confirmed"]):
                    continue
                q = anchor(to.box(t["mean"]))
                qin = [inside(z, q) for z in zones]
                for z, v in enumerate(qin):
                    occ[z] += v
                r = rec.get(t["id"])
                sides = [sign(orient(*g, *q)) for g in lines]
                if r is None:
                    rec[t["id"]] = {"anchor": q, "sides": sides, "inside": qin}
                    continue
                p = r["anchor"]
                for l, g in enumerate(lines):
                    stored, sq = r["sides"][l], sides[l]
                    if stored != 0 and sq == -stored and sign(orient(*g, *p)) * sq <= 0 and \
                            sign(orient(*p, *q, g[0], g[1])) * sign(orient(*p, *q, g[2], g[3])) <= 0:
                        tot["lines"][l, 0 if sq > 0 else 1] += 1
                        ev.append((LINE, l, sq, t["id"], t["cls"], q[0], q[1], st["frame"]))
                    if sq != 0:
                        r["sides"][l] = sq
                for z in range(len(zones)):
                    if qin[z] != r["inside"][z]:
                        tot["zones"][z, 0 if qin[z] else 1] += 1
                        ev.append((ENTRY if qin[z] else EXIT, z, 1 if qin[z] else -1, t["id"], t["cls"], q[0], q[1], st["frame"]))
                r["anchor"], r["inside"] = q, qin
            events.append([tuple(float(c) for c in e) for e in ev])
            occupancy.append(occ)
        return events, [len(e) for e in events], occupancy

    def records(self, s):
        """Stream s's records in the form yfv2_engine.Counter.records gives them for live tracks."""
        return {i: (r["anchor"], list(r["sides"]), sum(1 << z for z, v in enumerate(r["inside"]) if v)) for i, r in self.rec[s].items()}

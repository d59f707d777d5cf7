"""Scalar-Python restatement (test infrastructure) of the multi-stream tracker of yfv2_track_update (include/yfv2.h): ByteTrack's
three association stages, each solved by Crouse's shortest augmenting path, and its track lifecycle with a constant-velocity
Kalman filter in four decoupled 2x2 blocks.  Every value is a Python float and every operation one IEEE fp64 operation with one
rounding, in the order the contract writes it, so the kernel must match this bit for bit.  min / max are `a < b ? a : b` /
`a > b ? a : b`; a division by zero gives what IEEE gives (Python would raise).

The stage costs, the solver's sweeps and dual updates and the duplicate rule also exist as numpy float64 operations over whole
rows (np.where for min / max, never np.minimum / np.maximum, and IEEE division): the same operations on the same values, fast
enough for 1024 x 2048 stages with long augmenting paths.  Tracker uses those by default; Tracker(scalar=True) runs the
element-by-element form, and the tests hold the two equal."""
import math

import numpy as np

INF = math.inf
SP, SV = 1 / 20, 1 / 160
SP2, SV10 = 2 * SP, 10 * SV
STAGE2_THR, STAGE3_THR, DUP_IOU = 0.5, 0.7, 0.85
TRACKED, LOST = 1, 2
DEFAULTS = dict(high_thresh=0.5, low_thresh=0.1, new_thresh=0.6, match_thresh=0.8, max_age=30)


def mn(a, b):
    return a if a < b else b


def mx(a, b):
    return a if a > b else b


def div(a, b):
    if b == 0.0:
        if a != a or a == 0.0:
            return math.nan
        return math.copysign(INF, a) * math.copysign(1.0, b)
    return a / b


def iou(a, b):
    """IoU of boxes a (the track) and b, (x1, y1, x2, y2), without the +1."""
    iw = mx(0.0, mn(a[2], b[2]) - mx(a[0], b[0]))
    ih = mx(0.0, mn(a[3], b[3]) - mx(a[1], b[1]))
    inter = iw * ih
    aa = (a[2] - a[0]) * (a[3] - a[1])
    ab = (b[2] - b[0]) * (b[3] - b[1])
    return div(inter, (aa + ab) - inter)


def box(mean):
    h = mean[3]
    w = mean[2] * h
    x1 = mean[0] - w / 2
    y1 = mean[1] - h / 2
    return (x1, y1, x1 + w, y1 + h)


def measure(r):
    w = r[2] - r[0]
    h = r[3] - r[1]
    return (r[0] + w / 2, r[1] + h / 2, div(w, h), h)


def initiate(z):
    sp, sv = SP2 * z[3], SV10 * z[3]
    pos, vel = (sp, sp, 1e-2, sp), (sv, sv, 1e-5, sv)
    mean = list(z) + [0.0] * 4
    cov = []
    for k in range(4):
        cov += [pos[k] * pos[k], 0.0, vel[k] * vel[k]]
    return mean, cov


def predict(t):
    if t["state"] == LOST:
        t["mean"][7] = 0.0
    m, c = t["mean"], t["cov"]
    h = m[3]
    qp, qv = SP * h, SV * h
    qp, qv = qp * qp, qv * qv
    for k in range(4):
        m[k] = m[k] + m[k + 4]
        p, x, v = c[3 * k], c[3 * k + 1], c[3 * k + 2]
        tt = x + v
        c[3 * k] = ((p + x) + tt) + (1e-2 * 1e-2 if k == 2 else qp)
        c[3 * k + 1] = tt
        c[3 * k + 2] = v + (1e-5 * 1e-5 if k == 2 else qv)


def update(t, z):
    m, c = t["mean"], t["cov"]
    rp = SP * m[3]
    rp = rp * rp
    for k in range(4):
        p, x, v = c[3 * k], c[3 * k + 1], c[3 * k + 2]
        s = p + (1e-1 * 1e-1 if k == 2 else rp)
        k0, k1 = div(p, s), div(x, s)
        y = z[k] - m[k]
        m[k] = m[k] + k0 * y
        m[k + 4] = m[k + 4] + k1 * y
        c[3 * k] = p - k0 * p
        c[3 * k + 1] = x - k0 * x
        c[3 * k + 2] = v - k1 * x


NT = 128                  # threads per CTA of k_track.cu: solver column j belongs to thread j % NT, warp (j % NT) // 32


def argmin(shortest, sc):
    """The argmin of one path step, the kernel's rule: start from (+inf, no column) and take an unvisited column only when its
    shortest is strictly smaller, so the lowest column wins ties.  shortest is never NaN (it is only ever set by r < shortest),
    and the first step of a path sets every free column below +inf (see yfv2.h), so a step without a candidate is a broken
    contract: it raises."""
    best, bj = INF, -1
    for j in range(len(shortest)):
        if not sc[j] and shortest[j] < best:
            best, bj = shortest[j], j
    if bj < 0:
        raise AssertionError("argmin: no unvisited column below +inf")
    return best, bj


def crouse_scalar(C, nr, nc):
    """Crouse's shortest augmenting path on the nr x nc (nr <= nc) matrix C, rows in order, element by element.  Returns
    col4row."""
    u, v = [0.0] * nr, [0.0] * nc
    col4row, row4col = [-1] * nr, [-1] * nc
    for cur in range(nr):
        shortest, path, SC, SR = [INF] * nc, [-1] * nc, [False] * nc, []
        i, min_val, sink = cur, 0.0, -1
        while sink < 0:
            SR.append(i)
            Ci, ui = C[i], u[i]
            for j in range(nc):
                if SC[j]:
                    continue
                r = ((min_val + Ci[j]) - ui) - v[j]
                if r < shortest[j]:
                    shortest[j], path[j] = r, i
            min_val, bj = argmin(shortest, SC)
            SC[bj] = True
            if row4col[bj] < 0:
                sink = bj
            else:
                i = row4col[bj]
        u[cur] = u[cur] + min_val
        for i in SR:
            if i != cur:
                u[i] = u[i] + (min_val - shortest[col4row[i]])
        for j in range(nc):
            if SC[j]:
                v[j] = v[j] - (min_val - shortest[j])
        j = sink
        while True:
            i = path[j]
            row4col[j] = i
            col4row[i], j = j, col4row[i]
            if i == cur:
                break
    return col4row


def tie_kinds(cols):
    """Which owners a tie among solver columns `cols` spans: "thread" (two columns of one thread), "lane" (two threads of one
    warp), "warp" (two warps)."""
    own = np.asarray(cols) % NT
    kinds = set()
    if len(np.unique(own)) < len(own):
        kinds.add("thread")
    warps = own // 32
    for w in np.unique(warps):
        if len(np.unique(own[warps == w])) > 1:
            kinds.add("lane")
    if len(np.unique(warps)) > 1:
        kinds.add("warp")
    return kinds


def crouse(C, log=None):
    """crouse_scalar with each relaxation sweep and dual update as numpy float64 operations over the columns: the same IEEE
    operations on the same values.  C: float64 [nr, nc], nr <= nc.  log (a dict): steps of each row's path, the length of each
    augmenting path, the owner kinds of every tie the argmin met, and whether a dual left the finite numbers."""
    nr, nc = C.shape
    u, v = np.zeros(nr), np.zeros(nc)
    col4row, row4col = np.full(nr, -1), np.full(nc, -1)
    steps, plen, ties = [], [], set()
    with np.errstate(all="ignore"):
        for cur in range(nr):
            shortest, path, SC, SR = np.full(nc, INF), np.full(nc, -1), np.zeros(nc, bool), []
            i, min_val, sink = cur, 0.0, -1
            while sink < 0:
                SR.append(i)
                r = ((min_val + C[i]) - u[i]) - v
                better = (r < shortest) & ~SC
                shortest[better] = r[better]
                path[better] = i
                cand = np.where(SC, INF, shortest)
                min_val = float(cand.min())
                if not min_val < INF:
                    raise AssertionError("argmin: no unvisited column below +inf (row %d, step %d)" % (cur, len(SR)))
                tied = np.flatnonzero(cand == min_val)
                bj = int(tied[0])
                if len(tied) > 1:
                    ties |= tie_kinds(tied)
                SC[bj] = True
                if row4col[bj] < 0:
                    sink = bj
                else:
                    i = int(row4col[bj])
            u[cur] = u[cur] + min_val
            sr = np.asarray(SR[1:], int)
            u[sr] = u[sr] + (min_val - shortest[col4row[sr]])
            v[SC] = v[SC] - (min_val - shortest[SC])
            j, n = sink, 0
            while True:
                i = int(path[j])
                row4col[j] = i
                col4row[i], j = j, int(col4row[i])
                n += 1
                if i == cur:
                    break
            steps.append(len(SR))
            plen.append(n)
    if log is not None:
        log.update(steps=steps, plen=plen, ties=ties, nonfinite=not (np.isfinite(u).all() and np.isfinite(v).all()))
    return col4row.tolist()


def assign_scalar(cost, thr):
    """One association stage on cost[t][d] (tracks in ascending id x detections in row order): the reduction, the smaller side
    as rows, C = c - thr for allowed pairs (c < thr) else 0, Crouse, and the allowed assigned pairs.  Returns [(t, d)]."""
    nt = len(cost)
    nd = len(cost[0]) if nt else 0
    ok = [[cost[a][b] < thr for b in range(nd)] for a in range(nt)]
    rt = [a for a in range(nt) if any(ok[a])]
    rd = [b for b in range(nd) if any(ok[a][b] for a in range(nt))]
    if not rt:
        return []
    tr = len(rt) > len(rd)
    rows, cols = (rd, rt) if tr else (rt, rd)

    def pair(i, j):
        return (cols[j], rows[i]) if tr else (rows[i], cols[j])

    C = []
    for i in range(len(rows)):
        row = []
        for j in range(len(cols)):
            a, b = pair(i, j)
            row.append(cost[a][b] - thr if ok[a][b] else 0.0)
        C.append(row)
    col4row = crouse_scalar(C, len(rows), len(cols))
    out = []
    for i, j in enumerate(col4row):
        a, b = pair(i, j)
        if ok[a][b]:
            out.append((a, b))
    return out


def assign(cost, thr, log=None):
    """assign_scalar on a float64 [nt, nd] array (or nested lists).  log (a dict) gets the sizes before and after the reduction,
    the orientation tr (detections as rows) and what crouse logs."""
    cost = np.asarray(cost, np.float64)
    if cost.ndim != 2 or cost.size == 0:
        return []
    ok = cost < thr
    rt, rd = np.flatnonzero(ok.any(1)), np.flatnonzero(ok.any(0))
    if log is not None:
        log.update(nt=cost.shape[0], nd=cost.shape[1], ntr=len(rt), ndr=len(rd))
    if not len(rt):
        return []
    tr = len(rt) > len(rd)
    sub, oks = cost[np.ix_(rt, rd)], ok[np.ix_(rt, rd)]
    with np.errstate(all="ignore"):
        C = np.where(oks, sub - thr, 0.0)
    if tr:
        C = np.ascontiguousarray(C.T)
    if log is not None:
        log.update(tr=bool(tr), nrow=C.shape[0], ncol=C.shape[1])
    col4row = crouse(C, log)
    out = []
    for i, j in enumerate(col4row):
        a, b = (rt[j], rd[i]) if tr else (rt[i], rd[j])
        if ok[a, b]:
            out.append((int(a), int(b)))
    return out


def iou_matrix(A, B):
    """iou of every box of A [n, 4] (the tracks) with every box of B [m, 4], elementwise numpy with mn / mx as np.where and the
    division IEEE's (what div restates)."""
    def vmn(x, y):
        return np.where(x < y, x, y)

    def vmx(x, y):
        return np.where(x > y, x, y)

    a, b = A[:, None, :], B[None, :, :]
    with np.errstate(all="ignore"):
        iw = vmx(0.0, vmn(a[..., 2], b[..., 2]) - vmx(a[..., 0], b[..., 0]))
        ih = vmx(0.0, vmn(a[..., 3], b[..., 3]) - vmx(a[..., 1], b[..., 1]))
        inter = iw * ih
        aa = (a[..., 2] - a[..., 0]) * (a[..., 3] - a[..., 1])
        ab = (b[..., 2] - b[..., 0]) * (b[..., 3] - b[..., 1])
        return inter / ((aa + ab) - inter)


def stage_costs_scalar(tracks, dets, fused):
    return [[1.0 - (iou(t["box"], d["box"]) * d["conf"] if fused else iou(t["box"], d["box"])) for d in dets] for t in tracks]


def stage_costs(tracks, dets, fused):
    if not tracks or not dets:
        return np.zeros((len(tracks), len(dets)))
    q = iou_matrix(np.array([t["box"] for t in tracks], np.float64), np.array([d["box"] for d in dets], np.float64))
    with np.errstate(all="ignore"):
        return 1.0 - (q * np.array([d["conf"] for d in dets], np.float64) if fused else q)


def finite(v):
    return v == v and v not in (INF, -INF)


class Tracker:
    """S streams of at most K tracks, as the device state holds them."""

    def __init__(self, S, K, scalar=False, log=False, **params):
        """scalar: the element-by-element stage costs, solver and duplicate rule instead of the numpy ones.  log: keep in
        self.log one dict per association stage (what assign logs, with the stream, frame and stage) and per duplicate rule
        (the number of pairs)."""
        self.S, self.K = S, K
        self.scalar = scalar
        self.log = [] if log else None
        self.p = dict(DEFAULTS, **params)
        self.streams = [None] * S
        self.reset()

    def reset(self, streams=None):
        for s in (range(self.S) if streams is None else streams):
            self.streams[s] = {"frame": 0, "next_id": 1, "tracks": []}

    def update(self, dets, counts, streams=None):
        """dets: float64 [B, M, 6] (array-like), counts [B].  Returns (rows: B lists of 8-tuples, counts [B], dropped [B])."""
        B = len(dets)
        streams = list(range(B)) if streams is None else list(streams)
        rows, dropped = [], []
        for b, s in enumerate(streams):
            M = len(dets[b])
            n = min(max(int(counts[b]), 0), M)
            self._where = dict(stream=s)
            o, d = self._step(self.streams[s], [tuple(float(v) for v in dets[b][j]) for j in range(n)])
            rows.append(o)
            dropped.append(d)
        return rows, [len(r) for r in rows], dropped

    def _step(self, st, rows):
        p = self.p
        st["frame"] += 1
        frame = st["frame"]
        tracks = st["tracks"]
        for t in tracks:
            predict(t)
            t["box"] = box(t["mean"])
            t["match"] = None
        dets = []
        for j, r in enumerate(rows):
            if all(finite(v) for v in r) and r[2] > r[0] and r[3] > r[1] and r[4] > p["low_thresh"]:
                dets.append({"row": j, "box": r[:4], "conf": r[4], "cls": r[5], "high": r[4] > p["high_thresh"], "match": None})
        hi = [d for d in dets if d["high"]]
        lo = [d for d in dets if not d["high"]]
        kind = {id(t): (2 if t["state"] == LOST else (1 if t["confirmed"] else 0)) for t in tracks}

        def stage(k, ts, ds, fused, thr):
            if self.scalar:
                pairs = assign_scalar(stage_costs_scalar(ts, ds, fused), thr)
            else:
                lg = None if self.log is None else dict(self._where, frame=frame, stage=k, thr=thr)
                pairs = assign(stage_costs(ts, ds, fused), thr, lg)
                if lg is not None:
                    self.log.append(lg)
            for a, b in pairs:
                ts[a]["match"] = ds[b]
                ds[b]["match"] = ts[a]

        stage(1, [t for t in tracks if kind[id(t)] != 0], hi, True, p["match_thresh"])
        stage(2, [t for t in tracks if kind[id(t)] == 1 and t["match"] is None], lo, False, STAGE2_THR)
        stage(3, [t for t in tracks if kind[id(t)] == 0], [d for d in hi if d["match"] is None], True, STAGE3_THR)
        live = []
        for t in tracks:
            d = t["match"]
            if d is not None:
                update(t, measure(d["box"]))
                t.update(state=TRACKED, confirmed=1, score=d["conf"], cls=d["cls"], end_frame=frame, det_row=d["row"])
            elif kind[id(t)] == 1:
                t["state"] = LOST
            elif kind[id(t)] == 0:
                continue
            live.append(t)
        births = [d for d in hi if d["match"] is None and d["conf"] >= p["new_thresh"]]
        born = births[:max(self.K - len(live), 0)]
        for q, d in enumerate(born):
            mean, cov = initiate(measure(d["box"]))
            live.append({"id": st["next_id"] + q, "cls": d["cls"], "state": TRACKED, "confirmed": int(frame == 1), "start_frame": frame,
                         "end_frame": frame, "score": d["conf"], "det_row": d["row"], "mean": mean, "cov": cov})
        st["next_id"] += len(born)
        gone = set()
        for t in live:
            t["box"] = box(t["mean"])
            if t["state"] == LOST and frame - t["end_frame"] > p["max_age"]:
                gone.add(id(t))
        dup = set()
        tk = [t for t in live if t["state"] == TRACKED]
        lo = [t for t in live if t["state"] == LOST and id(t) not in gone]
        if self.scalar:
            over = [(a, b) for a in tk for b in lo if iou(a["box"], b["box"]) > DUP_IOU]
        else:
            if self.log is not None:
                self.log.append(dict(self._where, frame=frame, stage="dup", pairs=len(tk) * len(lo)))
            q = iou_matrix(np.array([t["box"] for t in tk], np.float64).reshape(-1, 4), np.array([t["box"] for t in lo], np.float64).reshape(-1, 4))
            over = [(tk[x], lo[y]) for x, y in zip(*np.nonzero(q > DUP_IOU))]
        for a, b in over:
            dup.add(id(b) if frame - a["start_frame"] > frame - b["start_frame"] else id(a))
        st["tracks"] = [t for t in live if id(t) not in gone and id(t) not in dup]
        out = [t["box"] + (t["score"], t["cls"], float(t["id"]), float(t["det_row"]))
               for t in st["tracks"] if t["state"] == TRACKED and t["confirmed"]]
        return out, len(births) - len(born)

    def tracks(self, s):
        """Stream s's state in the form yfv2_engine.Tracker.tracks returns."""
        st = self.streams[s]
        keys = ("id", "cls", "state", "confirmed", "start_frame", "end_frame", "score", "det_row")
        return {"frame": st["frame"], "next_id": st["next_id"],
                "tracks": [dict({k: t[k] for k in keys}, mean=list(t["mean"]), cov=list(t["cov"])) for t in st["tracks"]]}

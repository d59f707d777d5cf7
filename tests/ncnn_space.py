"""Inputs for the deploy post-process (yfv2_ncnn_post, the ncnn sample's predHandle + nmsHandle) that land on chosen sides of its
decisions, and the host-side restatement needed to check that they do.

Every case is one image: two channel-last head tensors out2 [H/16, W/16, 5A+C] and out3 [H/32, W/32, 5A+C] with the sample's
parameters, plus `claims`, the decisions it was built to reach.  `check(case)` asserts each claim from the restatement below
(candidate scores and categories, box corners, pair IoUs); nothing here runs the NMS itself, which is what the tests compare
between the device, oracle/ncnn_post.c and the reference's own compiled code.  Everything is numpy; nothing needs a GPU.

Boxes are placed exactly: with anchors (1, 1) and scale 1, a reg row (0.25 + k/2s, 0.25 + l/2s, n/2, m/2) of cell (x, y) at
stride s decodes to centre (sx + k, sy + l) and size (n², m²), so even n, m give integer corners.
"""
import numpy as np

f32 = np.float32
INT_MIN = -2147483648
NT = 256                  # threads of the ncnn CTA
CHUNK = 64                # candidates per suppression block
MAX_A = 8                 # kMaxA
MAX_C = 32767             # cates are stored as short
SMEM_CAP = 227 * 1024     # kSmemCap


def pow2_at_least(m, lo=64):
    p = lo
    while p < m:
        p <<= 1
    return p


def smem_bytes(M):
    """k_ncnn.cu ncnn_layout(s, nullptr, M, MCp): shared memory of one ncnn CTA for M candidate slots."""
    r16 = lambda b: (b + 15) & ~15  # noqa: E731
    b = pow2_at_least(M) * 8 + M * 16 + r16(M * 4) + r16(M * 2) * 2
    return b + CHUNK * 16 + CHUNK * 4 + r16(CHUNK * 2) + CHUNK * 8 + 32


def slots(A, H, W):
    return A * ((H // 16) * (W // 16) + (H // 32) * (W // 32))


def fits(A, H, W):
    M = slots(A, H, W)
    return M <= 0xFFFF and smem_bytes(M) <= SMEM_CAP


def largest_square(A):
    """(last accepted side, first refused side) of square inputs, sides multiples of 32."""
    s = 32
    while fits(A, s + 32, s + 32):
        s += 32
    return s, s + 32


# ---- restatement of predHandle (sample/ncnn/src/yolo-fastestv2.cpp:113-183) for the side checks --------------------------------

def corner(v):
    """double -> int of a box corner: truncation toward zero; NaN or a truncated value outside the int range gives INT_MIN
    (what the sample's `int = double` compiles to on x86-64, cvttsd2si)."""
    v = np.asarray(v, np.float64)
    t = np.trunc(np.where(np.isfinite(v), v, 0.0))
    ok = np.isfinite(v) & (t >= -2147483648.0) & (t <= 2147483647.0)
    return np.where(ok, t, INT_MIN).astype(np.int64)


def candidates(c, thresh=None):
    """Every candidate slot in push order (level, row, column, anchor): dict of arrays score (f32), cate, box [n,4] (int64, the
    int corners), order, passed (score > thresh) and the unconverted double corners `raw`."""
    A, C, H = c["A"], c["C"], c["H"]
    thresh = f32(c["thresh"] if thresh is None else thresh)
    sw, sh = scales(c)
    out = {k: [] for k in ("score", "cate", "raw")}
    for lv, o in enumerate((c["out2"], c["out3"])):
        h, w, _ = o.shape
        stride = H // h
        v = o.reshape(h * w, -1)
        ys, xs = np.divmod(np.arange(h * w), w)
        for b in range(A):
            with np.errstate(invalid="ignore", over="ignore"):
                cs = v[:, 5 * A:5 * A + C] * v[:, 4 * A + b:4 * A + b + 1]
            pos = np.where(cs > 0, cs, f32(0))                   # NaN > 0 is false: skipped as by the sample's strict '>'
            best = pos.max(1)
            cate = np.where(best > 0, (pos == best[:, None]).argmax(1), -1)
            out["score"].append(np.where(best > 0, best, f32(-1)).astype(f32))
            out["cate"].append(cate)
            r = v[:, 4 * b:4 * b + 4].astype(np.float64)
            with np.errstate(invalid="ignore", over="ignore"):
                bcx = ((r[:, 0] * 2.0 - 0.5 + xs) * stride).astype(f32).astype(np.float64)
                bcy = ((r[:, 1] * 2.0 - 0.5 + ys) * stride).astype(f32).astype(np.float64)
                bw = ((r[:, 2] * 2.0) * (r[:, 2] * 2.0) * np.float64(c["anchors"][(lv * A + b) * 2])).astype(f32).astype(np.float64)
                bh = ((r[:, 3] * 2.0) * (r[:, 3] * 2.0) * np.float64(c["anchors"][(lv * A + b) * 2 + 1])).astype(f32).astype(np.float64)
                raw = np.stack([(bcx - 0.5 * bw) * sw, (bcy - 0.5 * bh) * sh, (bcx + 0.5 * bw) * sw, (bcy + 0.5 * bh) * sh], 1)
            out["raw"].append(raw)
    # level-major, then cell, then anchor
    res = {}
    for k in out:
        per_lv = []
        for lv in range(2):
            blocks = out[k][lv * A:(lv + 1) * A]
            per_lv.append(np.stack(blocks, 1).reshape((-1,) + blocks[0].shape[1:]))
        res[k] = np.concatenate(per_lv)
    res["box"] = corner(res["raw"])
    res["order"] = np.arange(len(res["score"]))
    res["passed"] = res["score"] > thresh
    return res


def scales(c):
    """scaleW / scaleH of the sample (:189-190): float(src) / float(input) in fp32, used as double."""
    sw, sh = c["src"]
    return float(f32(sw) / f32(c["W"])), float(f32(sh) / f32(c["H"]))


def iou(a, b):
    """nmsHandle's IoU (:89-92) of two int boxes, fp32, with the int differences wrapping as they do on the device."""
    def d(u, v):
        return f32(np.int32((int(u) - int(v) + 2 ** 31) % 2 ** 32 - 2 ** 31))
    area = lambda t: d(t[2], t[0]) * d(t[3], t[1])  # noqa: E731
    ia = f32(0)
    if not (a[0] > b[2] or a[2] < b[0] or a[1] > b[3] or a[3] < b[1]):
        ia = d(min(a[2], b[2]), max(a[0], b[0])) * d(min(a[3], b[3]), max(a[1], b[1]))
    with np.errstate(invalid="ignore", divide="ignore"):
        return f32(ia / ((area(a) + area(b)) - ia))


def kept_count_bound(c):
    return int(candidates(c)["passed"].sum())


def max_out_edges(count):
    """max_out values around a kept count: one row, one row short, exactly the count, one row of padding."""
    return [1, count - 1, count, count + 1]


def push_order_ties(c):
    """Largest number of passing candidates that share one score (1 = no ties)."""
    s = candidates(c)
    s = s["score"][s["passed"]]
    if len(s) == 0:
        return 0
    _, n = np.unique(s.view(np.uint32), return_counts=True)
    return int(n.max())


def golden_ok(c):
    """The reference's std::sort is libstdc++'s introsort, an insertion sort (stable) up to 16 elements: its order equals push
    order whenever no score is shared or at most 16 candidates pass."""
    return push_order_ties(c) == 1 or kept_count_bound(c) <= 16


# ---- builders ------------------------------------------------------------------------------------------------------------

def blank(name, A=1, C=4, H=64, W=64, thresh=0.3, nms=0.25, src=None, anchors=None, **claims):
    """All objectness 0 (every score -1, no candidate above thresh >= -1); anchors (1, 1) unless given."""
    ch = 5 * A + C
    c = dict(name=name, A=A, C=C, H=H, W=W, thresh=f32(thresh), nms=f32(nms), src=src or (W, H),
             anchors=np.ones(4 * A, f32) if anchors is None else np.asarray(anchors, f32),
             out2=np.zeros((H // 16, W // 16, ch), f32), out3=np.zeros((H // 32, W // 32, ch), f32), claims=dict(claims))
    c["out2"][..., :4 * A] = 0.25
    c["out3"][..., :4 * A] = 0.25
    return c


def put(c, slot, score=None, cate=0, box=None, obj=1.0, cls=None, reg=None):
    """Writes candidate `slot` (push order) of level 0 or 1: either `score` (obj = score, class `cate` probability 1, the others
    0: score = 1 * obj exactly) or obj and the whole class row `cls`; and either an exact box (cx, cy, n, m) -> centre (cx, cy),
    size (n², m²) or raw reg values.  The class row belongs to the cell, shared by its A anchors."""
    A = c["A"]
    h2, w2 = c["out2"].shape[:2]
    lv, s = (0, slot) if slot < h2 * w2 * A else (1, slot - h2 * w2 * A)
    o = c["out2"] if lv == 0 else c["out3"]
    w = o.shape[1]
    cell, b = divmod(s, A)
    y, x = divmod(cell, w)
    v = o[y, x]
    v[4 * A + b] = obj
    if cls is not None:
        v[5 * A:] = cls
    elif score is not None:
        v[4 * A + b] = score
        v[5 * A:] = 0
        v[5 * A + cate] = 1
    if box is not None:
        assert c["anchors"][2 * (lv * A + b)] == 1 and c["anchors"][2 * (lv * A + b) + 1] == 1
        st = 16 << lv
        cx, cy, n, m = box
        v[4 * b:4 * b + 4] = (0.25 + (cx - st * x) / (2.0 * st), 0.25 + (cy - st * y) / (2.0 * st), n / 2.0, m / 2.0)
    if reg is not None:
        v[4 * b:4 * b + 4] = reg
    return c


def random_head(name, seed, A, C, H, W, thresh=None, nms=0.45, src=None, anchors=None, keep=0.3, classes=None, sparse=None,
                **claims):
    """sigmoid(reg) | sigmoid(obj) | softmax(cls) of seeded logits, built in float64 and rounded once; `classes` dominant classes
    make same-class overlaps, `sparse` = k leaves k random classes per cell non-zero (a softmax over k of the C classes).  thresh
    defaults to a value between two scores that passes about `keep` of the candidates."""
    rs = np.random.RandomState(seed)
    if anchors is None:
        anchors = (rs.uniform(8, 120, 4 * A)).astype(f32)
    c = blank(name, A, C, H, W, 0.0, nms, src, anchors, **claims)
    for o in (c["out2"], c["out3"]):
        h, w, _ = o.shape
        reg = 1.0 / (1.0 + np.exp(-rs.normal(0, 1.5, (h, w, 4 * A))))
        obj = 1.0 / (1.0 + np.exp(-rs.normal(-0.5, 2.0, (h, w, A))))
        lg = rs.normal(0, 2.0, (h, w, C))
        if classes:
            lg[..., :classes] += 5.0
        if sparse:
            off = np.ones((h, w, C), bool)
            for y in range(h):
                for x in range(w):
                    off[y, x, rs.choice(C, sparse, replace=False)] = False
            lg[off] = -np.inf
        e = np.exp(lg - lg.max(-1, keepdims=True))
        o[...] = np.concatenate([reg, obj, e / e.sum(-1, keepdims=True)], -1).astype(f32)
    s = np.sort(candidates(c, thresh=-2)["score"])
    if thresh is None:
        i = int(len(s) * (1 - keep))
        thresh = f32((float(s[i - 1]) + float(s[i])) / 2) if 0 < i < len(s) and s[i - 1] < s[i] else f32(0)
    c["thresh"] = f32(thresh)
    return c


def crowd(name, seed, n, A=3, C=3, H=352, W=352, nms=0.45, spread=60, **claims):
    """n passing candidates (unique scores, descending with push order shuffled) of C classes, boxes of 16..64 px crowded into a
    spread x spread square, so that same-class suppression is frequent; all other slots have obj 0."""
    rs = np.random.RandomState(seed)
    c = blank(name, A, C, H, W, 0.0, nms, **claims)
    M = slots(A, H, W)
    h2, w2 = H // 16, W // 16
    lvl0 = h2 * w2 * A
    assert n <= lvl0
    idx = np.sort(rs.choice(lvl0, n, replace=False))
    sc = (np.arange(n, 0, -1) / (n + 1.0)).astype(f32)[rs.permutation(n)]
    cell_cate = rs.randint(C, size=h2 * w2)                     # the class row is per cell
    for k, slot in enumerate(idx):
        n_w, n_h = 2 * rs.randint(2, 5, 2)
        put(c, int(slot), score=sc[k], cate=int(cell_cate[slot // A]),
            box=(100 + rs.randint(spread), 100 + rs.randint(spread), n_w, n_h))
    assert M > n
    return c


def lane_ties():
    """Equal cls*obj at classes k and k+32 / k+64 (other warp lanes), the rest smaller: the smaller index wins (strict '>' scan)."""
    c = blank("lane_ties", A=3, C=80, H=64, W=64, thresh=0.1, nms=0.5)
    pairs = [(3, 35), (3, 67), (31, 63), (0, 64), (13, 45), (47, 79), (5, 69), (16, 48)]
    for i, (k0, k1) in enumerate(pairs):
        cls = np.full(80, 0.001, f32)
        cls[k0] = cls[k1] = f32(0.3 + 0.05 * i)
        put(c, 3 * i, cls=cls, obj=f32(0.9), box=(20 + 20 * i, 30, 4, 6))
    # equal products from different factors: cls 0.5 * obj 0.8 == cls 0.8 * obj 0.5 is not reachable with one obj; instead the
    # same value in three lanes, the earliest lane last in the row
    cls = np.full(80, 0.002, f32); cls[[9, 41, 73]] = f32(0.45)
    put(c, 3 * 8 + 1, cls=cls, obj=f32(0.75), box=(40, 50, 8, 4))
    c["claims"]["cates"] = {3 * i: k0 for i, (k0, _) in enumerate(pairs)} | {25: 9}
    return c


def cases_all():
    """Every case of the suite (single images)."""
    cs = []
    # ---- geometry: anchors, classes and input shapes (random heads, some same-class crowding) ------------------------------
    for A, C, (H, W) in ((1, 80, (32, 32)), (2, 80, (64, 160)), (3, 8, (352, 352)), (4, 80, (640, 352)), (8, 80, (64, 160))):
        cs.append(random_head("geo_a%d_%dx%d" % (A, H, W), 100 + A, A, C, H, W, classes=2, geo=(A, C, H, W)))
    for C in (1, 2, 31, 32, 33, 80, 150, 1000):
        cs.append(random_head("geo_c%d" % C, 200 + C, 3, C, 64, 160, classes=min(C, 2), sparse=50 if C > 150 else None,
                              geo=(3, C, 64, 160)))
    cs.append(random_head("geo_c32767", 300, 1, MAX_C, 32, 32, keep=0.6, sparse=40, geo=(1, MAX_C, 32, 32)))
    cs.append(random_head("geo_src333x199", 301, 3, 3, 320, 352, src=(333, 199), classes=2, nonint_scale=True))

    # ---- category -----------------------------------------------------------------------------------------------------------
    cs.append(lane_ties())
    c = blank("all_nonpositive", A=1, C=33, H=64, W=32, thresh=-2.0, nms=0.5)    # 10 slots, all -1 / -1
    for s in range(10):
        sign = 1 if s % 3 else -1                                                  # cls <= 0 with obj > 0, or cls >= 0 with obj < 0
        put(c, s, cls=np.where(np.arange(33) % 2, f32(-0.25 * sign), f32(0)), obj=f32(0.5 * sign), box=(8 + 5 * s, 20, 2, 2))
    c["claims"].update(all_minus_one=True)
    cs.append(c)
    c = blank("obj_zero", A=2, C=5, H=32, W=32, thresh=-0.5, nms=0.5)
    for s in range(4):
        put(c, s, cls=np.full(5, 0.2, f32), obj=f32(0.0) if s % 2 else f32(0.6), box=(10 + 4 * s, 10, 2, 2))
    c["claims"].update(cates={0: 0, 1: -1, 2: 0, 3: -1})
    cs.append(c)

    # ---- threshold ------------------------------------------------------------------------------------------------------------
    base = [f32(0.61), f32(0.5), f32(0.37), f32(0.25)]
    for name, thr, kept in (("thr_at_score", f32(0.5), 1), ("thr_below_score", np.nextafter(f32(0.5), f32(-1)), 2)):
        c = blank(name, A=1, C=3, H=64, W=64, thresh=thr, nms=0.5)
        for s, sc in enumerate(base):
            put(c, s, score=sc, cate=s % 3, box=(10 + 12 * s, 20, 4, 4))
        c["claims"].update(passed=kept)
        cs.append(c)
    c = blank("thr_minus2", A=3, C=4, H=32, W=32, thresh=-2.0, nms=0.3)           # 15 slots: all pass, -1/-1 ones suppress each other
    for s in (0, 4, 9):
        put(c, s, score=f32(0.2 + 0.1 * s), cate=s % 4, box=(8 + 3 * s, 12, 4, 4))
    c["claims"].update(passed=15, minus_one=12)
    cs.append(c)
    c = blank("thr_minus2_spread", A=3, C=4, H=32, W=32, thresh=-2.0, nms=0.3)    # -1/-1 boxes apart: several survive
    for s in range(15):
        if s % 5 == 0:
            put(c, s, score=f32(0.3 + 0.02 * s), cate=1, box=(20, 20, 4, 4))
        else:
            put(c, s, obj=f32(0), box=(4 + 20 * (s % 3), 4 + 20 * (s // 5), 4, 4))
    c["claims"].update(passed=15, minus_one=12)
    cs.append(c)
    c = random_head("thr_one", 400, 3, 20, 64, 64, thresh=1.0)
    c["claims"].update(passed=0)
    cs.append(c)
    c = random_head("thr_zero", 401, 1, 3, 64, 64, thresh=0.0, nms=0.3)
    c["out2"][0, 0, 4] = 0.0                                                       # one cell with obj 0: score -1, not > 0
    c["claims"].update(zero_thresh=True)
    cs.append(c)

    # ---- boxes ---------------------------------------------------------------------------------------------------------------
    c = blank("trunc_negative", A=2, C=2, H=64, W=64, thresh=0.1, nms=0.5, src=(333, 199), anchors=[30, 20, 11, 7, 40, 50, 9, 13])
    rs = np.random.RandomState(500)
    for s in range(8):
        put(c, s, score=f32(0.9 - 0.05 * s), cate=(s // 2) % 2, reg=rs.uniform(0.0, 0.6, 4).astype(f32))
    # x1 = (bcx - 15) * 333/64 = -0.7 in column 0 (slot 8: row 1, anchor 0): reg x = (bcx/16 + 0.5) / 2, anchor 30, reg w 0.5
    sw = float(f32(333) / f32(64))
    put(c, 8, score=f32(0.3), cate=0, reg=[f32(((15 - 0.7 / sw) / 16 + 0.5) / 2), 0.3, 0.5, 0.5])
    c["claims"].update(truncates_to_zero=True, negative_fraction=True, nonint_scale=True)
    cs.append(c)
    c = blank("zero_area_identical", A=1, C=2, H=64, W=64, thresh=0.1, nms=0.3)
    put(c, 0, score=f32(0.9), cate=0, box=(20, 20, 0, 4))     # zero width
    put(c, 1, score=f32(0.8), cate=0, box=(20, 20, 0, 4))     # identical zero-area box: 0/0 IoU is NaN, not > thr: kept
    put(c, 2, score=f32(0.7), cate=1, box=(40, 40, 4, 4))
    put(c, 3, score=f32(0.6), cate=1, box=(40, 40, 4, 4))     # identical box of the same class: IoU 1, suppressed
    put(c, 4, score=f32(0.5), cate=0, box=(40, 40, 4, 4))     # identical box of another class: kept
    c["claims"].update(pairs={(0, 1): "nan", (2, 3): 1.0})
    cs.append(c)
    for nms in (0.0, 1.0, -0.1):
        c = blank("touch_nms%g" % nms, A=1, C=1, H=64, W=64, thresh=0.1, nms=nms)
        put(c, 0, score=f32(0.9), box=(20, 20, 2, 2))        # [18, 18, 22, 22]
        put(c, 1, score=f32(0.8), box=(24, 20, 2, 2))        # [22, 18, 26, 22]: x2 == x1', zero-width intersection
        put(c, 2, score=f32(0.7), box=(40, 20, 2, 2))        # [38, 18, 42, 22]: disjoint from both
        put(c, 3, score=f32(0.6), box=(20, 20, 4, 4))        # [12, 12, 28, 28] contains slots 0 and 1: IoU 1/16
        put(c, 4, score=f32(0.55), box=(40, 20, 2, 2))       # identical to slot 2: IoU exactly 1
        c["claims"].update(pairs={(0, 1): 0.0, (2, 4): 1.0}, touching=(0, 1), nms_edge=nms)
        cs.append(c)
    # IoU exactly nms_thresh (1/3 and 3/7 on integer boxes), and nms_thresh one fp32 step below / above it
    for q, (dx, n) in (("third", (8, 4)), ("3_7", (4, 4))):
        a = (40, 40, n, n)
        b = (40 + dx, 40, n, n)
        ia = iou(box_of(a), box_of(b))
        for side, thr in (("at", ia), ("below", np.nextafter(ia, f32(-1))), ("above", np.nextafter(ia, f32(2)))):
            c = blank("iou_%s_%s" % (q, side), A=1, C=1, H=96, W=96, thresh=0.1, nms=thr)
            put(c, 0, score=f32(0.9), box=a)
            put(c, 1, score=f32(0.8), box=b)
            c["claims"].update(pairs={(0, 1): float(ia)}, suppressed=(side == "below"))
            cs.append(c)

    # ---- chunks of 64 -----------------------------------------------------------------------------------------------------------
    for n in (1, 63, 64, 65, 128, 129):
        cs.append(crowd("chunk_%d" % n, 600 + n, n, count=n))
    c = blank("chain", A=1, C=2, H=352, W=352, thresh=0.05, nms=0.3)
    # 64 other-class boxes first, then A (score 0.99) kills B (chunk 1, IoU 1/3 > 0.3), B would kill C (IoU 1/3) but is dead
    for s in range(63):
        put(c, 10 + s, score=f32(0.98 - 0.001 * s), cate=1, box=(200 + 3 * s, 300, 2, 2))
    put(c, 0, score=f32(0.99), cate=0, box=(40, 40, 4, 4))        # A [32,32,48,48]
    put(c, 1, score=f32(0.5), cate=0, box=(48, 40, 4, 4))         # B [40,32,56,48]
    put(c, 2, score=f32(0.4), cate=0, box=(56, 40, 4, 4))         # C [48,32,64,48]: touches A
    c["claims"].update(pairs={(0, 1): 1 / 3, (1, 2): 1 / 3, (0, 2): 0.0}, chain=True)
    cs.append(c)
    cs.append(crowd("survivors_chunks", 700, 400, C=2, spread=200, nms=0.3, count=400))

    # ---- limits -----------------------------------------------------------------------------------------------------------------
    c = crowd("max_out", 800, 100, C=2, spread=120, nms=0.3)
    cs.append(c)

    # ---- non-finite values ------------------------------------------------------------------------------------------------------
    c = blank("nonfinite_box", A=2, C=2, H=64, W=64, thresh=0.1, nms=0.3, src=(128, 96))
    vals = [np.nan, np.inf, -np.inf]
    k = 0
    for s in range(6):
        reg = np.full(4, 0.3, f32)
        reg[s % 4] = vals[s % 3]
        put(c, s, score=f32(0.9 - 0.1 * s), cate=(s // 2) % 2, reg=reg)
        k += 1
    put(c, 6, score=f32(0.2), cate=0, reg=[0.3, 0.3, 0.5, 0.5])
    c["claims"].update(int_min=True)
    cs.append(c)
    c = blank("huge_box", A=1, C=2, H=64, W=64, thresh=0.1, nms=0.3, src=(256, 64))
    put(c, 0, score=f32(0.9), cate=0, reg=[0.3, 0.3, 1e6, 0.4])                  # width ~4e12: both x corners out of range
    put(c, 1, score=f32(0.8), cate=0, reg=[1e6, 0.3, 0.4, 0.4])                  # centre 1.3e8 * 4: x corners out of range
    put(c, 2, score=f32(0.7), cate=1, reg=[0.3, 1e6, 0.4, 0.4])                  # centre y 3.2e7: in range
    put(c, 3, score=f32(0.6), cate=1, reg=[0.3, -1e6, 0.4, 0.4])
    put(c, 4, score=f32(0.5), cate=1, reg=[16777000.0, 0.3, 59.0, 0.4])         # x1 in range, x2 past INT_MAX: x2 - x1 wraps
    put(c, 5, score=f32(0.45), cate=1, reg=[0.3, 0.3, 0.4, 0.4])
    c["claims"].update(int_min=True, mixed_corner=True)
    cs.append(c)
    c = blank("nan_scores", A=2, C=4, H=32, W=32, thresh=0.05, nms=0.4)
    put(c, 0, cls=np.array([0.2, np.nan, 0.5, 0.1], f32), obj=f32(0.9), box=(10, 10, 2, 2))    # NaN class skipped: cate 2
    put(c, 2, cls=np.array([0.2, 0.3, 0.5, 0.1], f32), obj=f32(np.nan), box=(14, 10, 2, 2))    # NaN obj: score -1
    put(c, 4, cls=np.array([np.nan, 0.7, 0.7, np.nan], f32), obj=f32(0.5), box=(20, 20, 2, 2))  # tie after NaN: cate 1
    put(c, 6, cls=np.array([np.inf, 0.1, 0.1, 0.1], f32), obj=f32(0.5), box=(24, 24, 2, 2))    # inf score
    c["claims"].update(cates={0: 2, 2: -1, 4: 1, 6: 0})
    cs.append(c)
    c = blank("src_out_of_range", A=1, C=2, H=32, W=64, thresh=0.1, nms=0.3, src=(2147483647, 1))
    for s in range(4):
        put(c, s, score=f32(0.8 - 0.1 * s), cate=s % 2, box=(50 + 6 * s, 10, 2, 2))      # x * 2^25: past INT_MAX from x = 64
    c["claims"].update(int_min=True, mixed_corner=True)
    cs.append(c)
    return cs


def box_of(b):
    cx, cy, n, m = b
    return (cx - n * n // 2, cy - m * m // 2, cx + n * n // 2, cy + m * m // 2)


def limit_cases():
    """The largest M whose shared memory fits, per A in (1, 3, 8), C = 1, every slot passing with a unique score (compared with
    the oracle on the GPU; refused sides are checked on the host)."""
    out = []
    for A in (1, 3, 8):
        side, _ = largest_square(A)
        c = blank("limit_a%d_%d" % (A, side), A=A, C=1, H=side, W=side, thresh=0.0, nms=0.4)
        rs = np.random.RandomState(900 + A)
        M = slots(A, side, side)
        sc = ((np.arange(M) + 1.0) / (M + 1.0)).astype(f32)[rs.permutation(M)]
        for o, n0 in ((c["out2"], 0), (c["out3"], c["out2"].shape[0] * c["out2"].shape[1] * A)):
            h, w, _ = o.shape
            o[..., 5 * A] = 1.0
            s = sc[n0:n0 + h * w * A].reshape(h, w, A)
            o[..., 4 * A:5 * A] = s                     # score = cls (1) * obj
            o[..., :4 * A] = rs.randint(13, 52, (h, w, 4 * A)) / f32(64)
        c["anchors"] = rs.uniform(8, 40, 4 * A).astype(f32)
        c["claims"].update(limit=(A, side), count=M)
        out.append(c)
    return out


def check(c):
    """Asserts every claim of case c from the restatement above; returns the candidates."""
    cand = candidates(c)
    cl = c["claims"]
    p = cand["passed"]
    if "geo" in cl:
        A, C, H, W = cl["geo"]
        assert (c["A"], c["C"], c["H"], c["W"]) == (A, C, H, W)
        assert 0 < p.sum() < len(p), c["name"]
    if "count" in cl or "passed" in cl:
        assert p.sum() == cl.get("count", cl.get("passed")), (c["name"], p.sum())
    if "cates" in cl:
        for s, k in cl["cates"].items():
            assert cand["cate"][s] == k, (c["name"], s, cand["cate"][s], k)
    if cl.get("all_minus_one"):
        assert (cand["score"] == -1).all() and (cand["cate"] == -1).all() and p.all()
    if "minus_one" in cl:
        assert ((cand["cate"] == -1) & p).sum() == cl["minus_one"]
    if cl.get("zero_thresh"):
        assert (cand["score"] == -1).any() and not p[cand["score"] == -1].any() and p.any()
    if cl.get("nonint_scale"):
        sw, sh = scales(c)
        assert sw != round(sw) and sh != round(sh)
    if cl.get("truncates_to_zero"):
        r = cand["raw"][p]
        assert ((r > -1) & (r < 0)).any(), "no corner in (-1, 0)"
    if cl.get("negative_fraction"):
        r = cand["raw"][p]
        assert ((r < -1) & (r != np.trunc(r))).any(), "no negative fractional corner"
    if "pairs" in cl:
        for (i, j), want in cl["pairs"].items():
            got = iou(cand["box"][i], cand["box"][j])
            assert (np.isnan(got) if want == "nan" else got == f32(want)), (c["name"], i, j, got, want)
    if "touching" in cl:
        i, j = cl["touching"]
        assert cand["box"][i][2] == cand["box"][j][0]
    if "suppressed" in cl:
        assert (iou(cand["box"][0], cand["box"][1]) > c["nms"]) == cl["suppressed"]
    if cl.get("int_min"):
        assert (cand["box"][p] == INT_MIN).any() and (np.isnan(cand["raw"][p]) | (np.abs(cand["raw"][p]) > 2 ** 31)).any()
    if cl.get("mixed_corner"):
        b = cand["box"][p]
        assert ((b[:, 0] != INT_MIN) & (b[:, 2] == INT_MIN)).any()
    if "limit" in cl:
        A, side = cl["limit"]
        assert fits(A, side, side) and not fits(A, side + 32, side + 32)
        assert len(np.unique(cand["score"])) == len(cand["score"])
    return cand

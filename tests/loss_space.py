"""Host-side restatement of the decisions build_target makes, and seeded loss cases that land on chosen sides of them.

build_target (reference utils/loss.py:53-124, csrc/k_loss.cu build_target_kernel) keeps a (target, anchor) pair when the largest
of w/aw, aw/w, h/ah, ah/h is below 2 (fp64); it adds the neighbour cell left / above / right / below of the target when the
fractional part of gx, gy, w - gx, h - gy is below 0.5 and the value above 1 (fp32); it truncates gxy - offset to a cell and
clamps that cell into the grid before tbox = gxy - cell.  `decide` restates those decisions in the reference's dtypes and `rows`
builds the matched rows from them in the reference's order (offset-major, then anchor, then target).

Every case records which side of each decision its targets were built for, and `check_sides` asserts it on the host.  The CIoU
cases set every box logit to 0, so each predicted box is (0.5, 0.5, aw, ah) exactly, and record which fp64 edges of the predicted
and target boxes coincide.  `ciou_grad` is the hand-written reverse mode of loss_rows_kernel in fp64, with a chosen share of a
min / max term at a tie.  Everything here is numpy; nothing needs a GPU.
"""
import hashlib
import math

import numpy as np

f32, f64 = np.float32, np.float64
OFFSETS = ((0.0, 0.0), (0.5, 0.0), (0.0, 0.5), (-0.5, 0.0), (0.0, -0.5))   # loss.py:67-71 times g = 0.5
CHUNK = 1024                                                                # candidates per pass of build_target_kernel
COCO_ANCHORS = [12.64, 19.39, 37.88, 51.48, 55.71, 138.31, 126.91, 78.23, 131.57, 214.55, 279.92, 258.87]
EDGES = ("x1", "x2", "y1", "y2")
T, F = True, False


def up(x):
    return np.nextafter(f32(x), f32(np.inf))


def down(x):
    return np.nextafter(f32(x), f32(-np.inf))


def levels(H, W):
    return ((H // 16, W // 16), (H // 32, W // 32))


def cfg_of(case):
    """The dict load_datafile returns, for the keys compute_loss reads."""
    return {"model_name": case["name"], "classes": case["C"], "width": case["W"], "height": case["H"],
            "anchor_num": case["A"], "anchors": list(case["anchors"])}


# ---- build_target, restated ---------------------------------------------------------------------------------------------------
def decide(case, lv):
    """build_target's decisions at level lv: gxy, gwh and gxi (fp32, [nt,2]), the anchors in grid units (fp64 [A,2]), the largest
    anchor ratio (fp64 [A,nt]), the ratio test [A,nt] and the five offset flags [5,nt] (centre, j, k, l, m)."""
    H, W, A = case["H"], case["W"], case["A"]
    h, w = levels(H, W)[lv]
    t = case["targets"]
    g = t[:, 2:6] * np.array([w, h, w, h], f32)                            # gt = targets * gain, fp32 (loss.py:89)
    a_cfg = np.array(case["anchors"], f64).reshape(2, A, 2)[lv] / (W / w)  # anchors / stride, fp64 (loss.py:81,84)
    r = g[None, :, 2:4].astype(f64) / a_cfg[:, None, :]                    # fp64 (loss.py:93)
    ratio = np.maximum(r, 1.0 / r).max(2) if len(t) else np.zeros((A, 0))
    gxy = g[:, 0:2]
    gxi = np.array([w, h], f32) - gxy                                      # loss.py:100
    near = (np.fmod(gxy, f32(1)) < f32(0.5)) & (gxy > f32(1))              # loss.py:101
    far = (np.fmod(gxi, f32(1)) < f32(0.5)) & (gxi > f32(1))               # loss.py:102
    flags = np.stack([np.ones(len(t), bool), near[:, 0], near[:, 1], far[:, 0], far[:, 1]])
    return dict(h=h, w=w, gxy=gxy, gwh=g[:, 2:4], gxi=gxi, a_cfg=a_cfg, ratio=ratio, accept=ratio < 2, flags=flags)


def candidates(case, lv):
    """[5, A, nt] mask of the kept candidates; flattened in C order it is build_target_kernel's candidate index."""
    d = decide(case, lv)
    return d["accept"][None] & d["flags"][:, None, :]


def rows(case, lv):
    """The matched rows of level lv in the reference's order: b, a, gj, gi, cls (int64), tbox [m,4] fp32, anch [m,2] fp64, and
    per row the offset o, the target t and the cell before the clamp (gij_raw [m,2], x then y)."""
    d = decide(case, lv)
    t = case["targets"]
    o, a, ti = np.nonzero(candidates(case, lv))
    gxy = d["gxy"][ti]
    gij_raw = (gxy - np.array(OFFSETS, f32)[o]).astype(np.int64)           # fp32 subtract, .long() truncates (loss.py:114)
    gi = np.clip(gij_raw[:, 0], 0, d["w"] - 1)                             # clamp_ before tbox (loss.py:119-120)
    gj = np.clip(gij_raw[:, 1], 0, d["h"] - 1)
    tbox = np.concatenate([gxy - np.stack([gi, gj], 1).astype(f32), d["gwh"][ti]], 1).astype(f32)
    return dict(b=t[ti, 0].astype(np.int64), a=a.astype(np.int64), gj=gj, gi=gi, cls=t[ti, 1].astype(np.int64), tbox=tbox,
                anch=d["a_cfg"][a], o=o, t=ti, gij_raw=gij_raw)


def find_row(case, lv, t, o, a):
    r = rows(case, lv)
    k = np.nonzero((r["t"] == t) & (r["o"] == o) & (r["a"] == a))[0]
    assert len(k) == 1, (case["name"], lv, t, o, a)
    return r, int(k[0])


# ---- CIoU at a matched row ------------------------------------------------------------------------------------------------------
def edges(x, y, w, h):
    return {"x1": x - w / 2, "x2": x + w / 2, "y1": y - h / 2, "y2": y + h / 2}


def box_relation(p, t):
    """How the fp64 predicted box p and target box t (x, y, w, h) meet: the tied edges, iw_raw / ih_raw (intersection before the
    clamp) and whether the boxes are identical."""
    b1 = edges(*map(float, p))
    tx, ty, tw, th = (f32(v) for v in t)                                    # tbox is fp32: so are its corners (loss.py:19-20)
    b2 = {k: float(v) for k, v in edges(tx, ty, tw, th).items()}
    iw = min(b1["x2"], b2["x2"]) - max(b1["x1"], b2["x1"])
    ih = min(b1["y2"], b2["y2"]) - max(b1["y1"], b2["y1"])
    tied = {e for e in EDGES if b1[e] == b2[e]}
    return {"tied": tied, "iw_raw": iw, "ih_raw": ih, "identical": tied == set(EDGES)}


def row_relation(case, lv, t, o, a):
    """box_relation of one matched row in a case whose box logits are all 0 (predicted box (0.5, 0.5, aw, ah) exactly)."""
    assert all(not p.any() for p in (case["preds"][0], case["preds"][3])), case["name"]
    r, k = find_row(case, lv, t, o, a)
    aw, ah = r["anch"][k]
    return box_relation((0.5, 0.5, aw, ah), r["tbox"][k])


def ciou_grad(p, t, tie_share):
    """d(ciou)/d(px, py, pw, ph) by loss_rows_kernel's hand-written reverse mode, all in fp64 (the kernel takes the target box's
    own terms in fp32, as the reference does).  At an exact tie of a min / max the predicted box gets `tie_share` of the term:
    torch.min / torch.max give it 0.5; 0 is the strict comparison alone.  A predicted height of 0 gives NaN, as in autograd."""
    px, py, pw, ph = map(float, p)
    b1, b2 = edges(px, py, pw, ph), edges(*map(float, t))

    def dmin(a, b):
        return 1.0 if a < b else (tie_share if a == b else 0.0)

    def dmax(a, b):
        return 1.0 if a > b else (tie_share if a == b else 0.0)
    iw_raw = min(b1["x2"], b2["x2"]) - max(b1["x1"], b2["x1"])
    ih_raw = min(b1["y2"], b2["y2"]) - max(b1["y1"], b2["y1"])
    iw, ih = max(iw_raw, 0.0), max(ih_raw, 0.0)
    inter = iw * ih
    w1, h1 = b1["x2"] - b1["x1"], b1["y2"] - b1["y1"]
    w2, h2 = b2["x2"] - b2["x1"], b2["y2"] - b2["y1"]
    uni = (w1 * h1 + 1e-16) + w2 * h2 - inter
    iou = inter / uni
    cw = max(b1["x2"], b2["x2"]) - min(b1["x1"], b2["x1"])
    ch = max(b1["y2"], b2["y2"]) - min(b1["y1"], b2["y1"])
    c2 = cw * cw + ch * ch + 1e-16
    sx = (b2["x1"] + b2["x2"]) - (b1["x1"] + b1["x2"])
    sy = (b2["y1"] + b2["y2"]) - (b1["y1"] + b1["y2"])
    rho2 = sx * sx / 4 + sy * sy / 4
    x1 = w1 / h1 if h1 else (math.inf if w1 else math.nan)
    D = math.atan(w2 / h2) - math.atan(x1)
    v = 4 / math.pi ** 2 * D * D
    alpha = v / (1 - iou + v)
    g_inter, g_u0, g_c2, g_rho, g_v = 1 / uni + inter / (uni * uni), -inter / (uni * uni), rho2 / (c2 * c2), -1 / c2, -alpha
    g = dict.fromkeys(EDGES, 0.0)
    if iw_raw >= 0:
        g["x2"] += g_inter * ih * dmin(b1["x2"], b2["x2"]); g["x1"] -= g_inter * ih * dmax(b1["x1"], b2["x1"])
    if ih_raw >= 0:
        g["y2"] += g_inter * iw * dmin(b1["y2"], b2["y2"]); g["y1"] -= g_inter * iw * dmax(b1["y1"], b2["y1"])
    g["x2"] += g_u0 * h1; g["x1"] -= g_u0 * h1; g["y2"] += g_u0 * w1; g["y1"] -= g_u0 * w1
    g["x2"] += g_c2 * 2 * cw * dmax(b1["x2"], b2["x2"]); g["x1"] -= g_c2 * 2 * cw * dmin(b1["x1"], b2["x1"])
    g["y2"] += g_c2 * 2 * ch * dmax(b1["y2"], b2["y2"]); g["y1"] -= g_c2 * 2 * ch * dmin(b1["y1"], b2["y1"])
    for e in ("x1", "x2"):
        g[e] += g_rho * (-sx / 2)
    for e in ("y1", "y2"):
        g[e] += g_rho * (-sy / 2)
    g_at = -g_v * (8 / math.pi ** 2) * D / (1 + x1 * x1)
    g_w1 = g_at / h1 if h1 else math.nan
    g_h1 = -g_at * (x1 / h1) if h1 else math.nan
    g["x2"] += g_w1; g["x1"] -= g_w1; g["y2"] += g_h1; g["y1"] -= g_h1
    return np.array([g["x1"] + g["x2"], g["y1"] + g["y2"], (g["x2"] - g["x1"]) / 2, (g["y2"] - g["y1"]) / 2])


# The three tie rows worked out when the tie bug was found: pred (x, y, w, h) -> target, d(ciou)/d(px, py, pw, ph) of torch's
# autograd and of the strict comparisons, to four decimals.
TIE_TABLE = [
    ((.5, .5, 2, 1.5), (.5, .6, 2, 1.2), {"x1", "x2"}, [0, .032, -.0391, -.5331], [0, .032, -.3996, -.5331]),
    ((.5, .5, 2, 1.5), (.75, .5, 2.5, 1.2), {"x1"}, [.3344, 0, .1417, -.3700], [.6144, 0, .0017, -.3700]),
    ((.5, .5, 2, 1.5), (.6, .5, 2.5, 1.5), {"y1", "y2"}, [.0235, 0, .4004, .0530], [.0235, 0, .4004, -.4272]),
]


# ---- inputs ------------------------------------------------------------------------------------------------------------------
def draw(rs, kind, shape):
    """Logits of one head tensor: 'randn', ('scale', s), ('const', v), ('choice', values) or ('uniform', lo, hi)."""
    if kind == "randn":
        return rs.randn(*shape).astype(f32)
    if kind[0] == "scale":
        return (kind[1] * rs.randn(*shape)).astype(f32)
    if kind[0] == "const":
        return np.full(shape, kind[1], f32)
    if kind[0] == "choice":
        return rs.choice(np.array(kind[1], f32), shape).astype(f32)
    return rs.uniform(kind[1], kind[2], shape).astype(f32)


def head_logits(seed, N, H, W, A, C, reg="randn", obj="randn", cls=("scale", 2.0)):
    rs = np.random.RandomState(seed)
    out = []
    for h, w in levels(H, W):
        out += [draw(rs, reg, (N, 4 * A, h, w)), draw(rs, obj, (N, A, h, w)), draw(rs, cls, (N, C, h, w))]
    return tuple(out)


def random_targets(rs, n, N, C, wh=(0.02, 0.52), images=None):
    """n rows (image, class, x, y, w, h), normalised, every index in range."""
    b = rs.choice(images, n) if images is not None else rs.randint(0, N, n)
    return np.stack([b, rs.randint(0, C, n), rs.rand(n), rs.rand(n), rs.uniform(wh[0], wh[1], n), rs.uniform(wh[0], wh[1], n)],
                    1).astype(f32).reshape(-1, 6)


def grid_target(b, c, gx, gy, gw, gh, w, h):
    """A target row given in grid units of a level whose w and h are powers of two, so that gt = targets * gain gives back the
    same fp32 values."""
    return [b, c, f32(gx) / f32(w), f32(gy) / f32(h), f32(gw) / f32(w), f32(gh) / f32(h)]


def make(name, N, H, W, A, C, anchors, targets, seed, golden=True, sides=(), ties=(), checks=(), **logits):
    targets = np.asarray(targets, f32).reshape(-1, 6)
    case = dict(name=name, N=N, H=H, W=W, A=A, C=C, anchors=[float(v) for v in anchors], targets=targets,
                preds=head_logits(seed, N, H, W, A, C, **logits), golden=golden, sides=list(sides), ties=list(ties),
                checks=list(checks))
    assert len(case["anchors"]) == 4 * A
    return case


def input_digest(case):
    """SHA-256 of a case's targets and logits: the goldens store it to catch a changed builder."""
    h = hashlib.sha256(case["targets"].tobytes())
    for p in case["preds"]:
        h.update(np.ascontiguousarray(p).tobytes())
    return np.frombuffer(h.digest(), np.uint8)


# ---- the cases ----------------------------------------------------------------------------------------------------------------
SQ32 = [32, 32, 32, 32]                  # one 32-px anchor per level: 2.0 grid cells at stride 16, 1.0 at stride 32


def case_ratio():
    """The ratio test at exactly 2 (rejected) and one fp32 step inside (kept), on the w / aw and the aw / w side, for w and h.
    At 512x512 level 0 has a 32-wide grid (aw = 2) and level 1 a 16-wide one (aw = 1), so both levels see the same ratios."""
    tg, sides = [], []
    for i, (v, keep) in enumerate([(4.0, False), (down(4.0), True), (1.0, False), (up(1.0), True)]):
        tg.append(grid_target(0, 1, 9.25 + 2 * i, 9.25, v, 2.0, 32, 32))
        tg.append(grid_target(0, 0, 20.75, 9.25 + 2 * i, 2.0, v, 32, 32))
        for lv in (0, 1):
            sides += [(lv, 2 * i, 0, {"accept": keep}), (lv, 2 * i + 1, 0, {"accept": keep})]
    return make("ratio", 1, 512, 512, 1, 2, SQ32, tg, 501, sides=sides)


def case_offsets():
    """The neighbour-cell tests on both sides of each boundary: frac(gx) exactly 0.5 and just below, gx exactly 1 and just above,
    w - gx exactly 1 and just above, frac(w - gx) exactly 0.5 and just below; the same for y.  The other coordinate is k + 0.5,
    where neither neighbour test passes."""
    xs = [(5.5, F, F), (down(5.5), T, F), (1.0, F, T), (up(1.0), T, T), (31.0, T, F), (down(31.0), F, T), (26.5, F, F),
          (up(26.5), F, T)]
    tg, sides = [], []
    for i, (v, near, far) in enumerate(xs):
        tg.append(grid_target(0, 0, v, 10.5, 2.0, 2.0, 32, 32))
        tg.append(grid_target(0, 1, 10.5, v, 2.0, 2.0, 32, 32))
        sides.append((0, 2 * i, 0, {"accept": True, "j": near, "l": far, "k": False, "m": False}))
        sides.append((0, 2 * i + 1, 0, {"accept": True, "k": near, "m": far, "j": False, "l": False}))
    # gx - 0.5 one step below an integer truncates to the cell below: tbox x is 1.5 - 2^-21, and w - gx one step above 1 gives
    # the right neighbour with tbox x = -0.5 + 2^-19
    checks = [("trunc below 5", lambda c: _row(c, 0, 2, 1)["gi"] == 4 and _row(c, 0, 2, 1)["tbox"][0] == f32(1.5) - f32(2 ** -21)),
              ("right of 26.5+", lambda c: _row(c, 0, 14, 3)["gi"] == 27 and _row(c, 0, 14, 3)["tbox"][0] == f32(-0.5) + f32(2 ** -19))]
    return make("offsets", 1, 512, 512, 1, 2, SQ32, tg, 502, sides=sides, checks=checks)


def _row(case, lv, t, o, a=0):
    r, k = find_row(case, lv, t, o, a)
    return {key: r[key][k] for key in ("b", "a", "gj", "gi", "cls", "tbox", "gij_raw")}


ANCH_64x96 = [16, 16, 32, 24, 32, 32, 64, 64]


def case_borders():
    """x or y exactly 0 or 1 on a 64x96 input (H != W; a 4x6 and a 2x3 grid), two anchors, one class (no CE term), targets on
    the last image: a coordinate of 1 truncates to the cell past the grid and is clamped back, so tbox is exactly 1."""
    xy = [(0, 0), (1, 1), (0, 1), (1, 0), (1, 0.5), (0.5, 0), (0.5, 1)]
    tg = [[1, 0, x, y, 0.3, 0.3] for x, y in xy]
    checks = []
    for i, (x, y) in enumerate(xy):
        for lv in (0, 1):
            checks.append(("border %d lv%d" % (i, lv), lambda c, i=i, lv=lv, x=x, y=y: _border_ok(c, lv, i, x, y)))
    return make("borders", 2, 64, 96, 2, 1, ANCH_64x96, tg, 503, checks=checks)


def _border_ok(case, lv, t, x, y):
    r = rows(case, lv)
    h, w = levels(case["H"], case["W"])[lv]
    k = np.nonzero((r["t"] == t) & (r["o"] == 0))[0]
    if not len(k):
        return False
    k = k[0]
    ok = True
    for v, n, c in ((x, w, 0), (y, h, 1)):
        if v == 1:
            ok &= r["gij_raw"][k, c] == n and r["tbox"][k, c] == f32(1)      # clamped: tbox component exactly 1
        elif v == 0:
            ok &= r["gij_raw"][k, c] == 0 and r["tbox"][k, c] == f32(0)
    return bool(ok)


def case_empty():
    return make("empty", 2, 64, 96, 2, 2, ANCH_64x96, np.zeros((0, 6), f32), 504)


SMALL_ANCH = [8, 8, 12, 16, 20, 14, 16, 16, 24, 32, 32, 24]   # rows at level 1 of a 32x32 or 64x64 input too


def case_tiny32():
    """32x32: level 1 is a single cell, level 0 a 2x2 grid; 80 classes."""
    rs = np.random.RandomState(505)
    tg = np.concatenate([random_targets(rs, 9, 2, 80, wh=(0.2, 1.0)), [[1, 79, 1, 1, 0.5, 0.5], [1, 3, 0, 0, 0.9, 0.9]]])
    return make("tiny32", 2, 32, 32, 3, 80, SMALL_ANCH, tg.astype(f32), 506, checks=[("level 1 rows", lambda c: len(rows(c, 1)["b"]) > 0)])


def case_reject_level1():
    """Every target kept at level 0 (aw = 2) and rejected at level 1 (aw = 4), which then has no rows."""
    rs = np.random.RandomState(507)
    tg = random_targets(rs, 12, 2, 2, wh=(1.1 / 22, 3.9 / 22))
    sides = [(lv, t, 0, {"accept": lv == 0}) for t in range(12) for lv in (0, 1)]
    return make("reject_level1", 2, 352, 352, 1, 2, [32, 32, 128, 128], tg, 508, sides=sides)


def case_reject_all():
    """Targets far larger than every anchor: no rows at either level although nt > 0."""
    rs = np.random.RandomState(509)
    tg = random_targets(rs, 5, 1, 80, wh=(0.3, 0.6))
    sides = [(lv, t, a, {"accept": False}) for t in range(5) for a in range(2) for lv in (0, 1)]
    return make("reject_all", 1, 352, 352, 2, 80, [4, 4, 6, 6, 4, 4, 6, 6], tg, 510, sides=sides)


ANCH5 = [24, 24, 28, 20, 20, 28, 32, 32, 26, 26] * 2


def case_chunk(A, nt):
    """5*A*nt candidates around the 1024-candidate passes of the ordered compaction.  The last target sits on an interior grid
    point of level 0 with a box every anchor keeps, so the last candidate (offset m, anchor A-1) is a row."""
    rs = np.random.RandomState(511 + 7 * A + nt)
    tg = random_targets(rs, nt - 1, 4, 3, wh=(0.02, 0.2))
    tg = np.concatenate([tg, [[3, 2, 0.5, 0.5, 1.6 / 22, 1.6 / 22]]]).astype(f32)
    total = 5 * A * nt
    checks = [("last candidate kept", lambda c: bool(candidates(c, 0).reshape(-1)[total - 1])),
              ("rows on both sides of a pass boundary",
               lambda c: total < CHUNK or bool(candidates(c, 0).reshape(-1)[:CHUNK].any() and candidates(c, 0).reshape(-1)[CHUNK:].any()))]
    return make("chunk_%d" % total + ("_a%d" % A if A > 1 else ""), 4, 352, 352, A, 3, (ANCH5[:2 * A] * 2), tg, 512 + nt,
                checks=checks)


def case_same_cell():
    """Identical target rows, and different targets in the same (image, anchor, cell) or the same class cell: several rows add
    into one cell of the gradient and set one obj target."""
    rs = np.random.RandomState(513)
    tg = random_targets(rs, 10, 2, 80).tolist()
    tg += [tg[0], tg[0], tg[3]]                                    # identical rows
    tg += [[1, 5, 0.40, 0.40, 0.10, 0.12], [1, 7, 0.40, 0.40, 0.11, 0.10], [1, 9, 0.41, 0.41, 0.2, 0.2]]   # same cells

    def shared(c):
        r = rows(c, 0)
        key = r["b"] * 10 ** 6 + r["a"] * 10 ** 4 + r["gj"] * 100 + r["gi"]
        cls_key = r["b"] * 10 ** 4 + r["gj"] * 100 + r["gi"]
        dup = len(np.unique(key)) < len(key)
        cls_dup = any(len(np.unique(r["a"][cls_key == k])) > 1 for k in np.unique(cls_key))
        return dup and cls_dup
    return make("same_cell", 2, 352, 352, 3, 80, COCO_ANCHORS, tg, 514, checks=[("shared cells", shared)])


def case_saturated():
    """Saturated logits: obj +-20 / +-100, classes spread over +-80, box logits +-30 (the sigmoid is 0 or 1 in fp32)."""
    rs = np.random.RandomState(515)
    return make("saturated", 2, 352, 352, 3, 80, COCO_ANCHORS, random_targets(rs, 14, 2, 80), 516,
                obj=("choice", [-100.0, -20.0, 20.0, 100.0]), cls=("uniform", -80.0, 80.0),
                reg=("choice", [-30.0, -2.0, 0.0, 1.0, 30.0]))


def case_cls_tied():
    """150 classes, every class logit exactly equal."""
    rs = np.random.RandomState(517)
    return make("cls_tied", 1, 352, 352, 3, 150, COCO_ANCHORS, random_targets(rs, 8, 1, 150), 518, cls=("const", 1.25))


def case_a8_c150():
    rs = np.random.RandomState(519)
    anchors = list(np.round(rs.uniform(6, 60, 32), 2))
    return make("a8_c150", 2, 64, 64, 8, 150, anchors, random_targets(rs, 12, 2, 150, wh=(0.05, 0.6)), 520)


def case_n64():
    """Batch 64 with targets on the first and the last image."""
    rs = np.random.RandomState(521)
    return make("n64", 64, 64, 64, 3, 2, SMALL_ANCH, random_targets(rs, 10, 64, 2, wh=(0.1, 0.8), images=[0, 63]), 522)


TIE_ANCH = [32, 24, 8, 8, 32, 24, 8, 8]   # (2, 1.5) and (0.5, 0.5) grid cells at stride 16; (1, 0.75) and (0.25, 0.25) at 32


def case_ciou_ties():
    """Box logits 0, so the predicted box is (0.5, 0.5, aw, ah) exactly, and 512x512 grids, so tbox is exact: the three tie rows of
    TIE_TABLE, both x edges tied while the boxes are disjoint in y (the enclosing box alone routes them), touching boxes
    (iw_raw == 0, where the clamp passes its gradient) and disjoint boxes."""
    tg = [grid_target(0, 0, 3.5, 3.6, 2.0, 1.2, 32, 32),          # (.5, .6, 2, 1.2): both x edges
          grid_target(0, 1, 7.75, 7.5, 2.5, 1.2, 32, 32),         # (.75, .5, 2.5, 1.2): left edge
          grid_target(0, 0, 11.6, 11.5, 2.5, 1.5, 32, 32),        # (.6, .5, 2.5, 1.5): both y edges
          grid_target(0, 1, 5.5, 5.25, 1.0, 0.4, 16, 16),         # level 1, k row: x edges tied, y disjoint
          grid_target(0, 0, 6.0, 20.5, 0.5, 0.6, 32, 32),         # anchor 1: touching on both sides
          grid_target(0, 1, 14.0, 24.5, 0.3, 0.6, 32, 32)]        # anchor 1: disjoint in x
    ties = [(0, 0, 0, 0, {"tied": {"x1", "x2"}}), (0, 1, 0, 0, {"tied": {"x1"}}), (0, 2, 0, 0, {"tied": {"y1", "y2"}}),
            (1, 3, 2, 0, {"tied": {"x1", "x2"}, "ih_neg": True}),
            (0, 4, 0, 1, {"tied": set(), "iw_zero": True}), (0, 4, 1, 1, {"tied": set(), "iw_zero": True}),
            (0, 5, 1, 1, {"tied": set(), "iw_neg": True})]
    return make("ciou_ties", 1, 512, 512, 2, 2, TIE_ANCH, tg, 523, ties=ties, reg=("const", 0.0))


def case_ciou_identical():
    """A predicted box identical to its target.  With fp64 target corners D = atan(w2/h2) - atan(w1/h1) would be exactly 0 and
    alpha 0/0; the reference's target box is fp32, its atan(w2/h2) too, so D is an fp32 rounding error, alpha is 1 and the row's
    CIoU is 1 - v: finite."""
    tg = [grid_target(0, 1, 4.5, 4.5, 2.0, 1.5, 32, 32), grid_target(0, 0, 17.3, 9.8, 1.7, 1.1, 32, 32)]
    return make("ciou_identical", 1, 512, 512, 2, 2, TIE_ANCH, tg, 524, ties=[(0, 0, 0, 0, {"identical": True})],
                reg=("const", 0.0))


def case_ciou_nan():
    """A predicted box of zero size: box logits -200 for w and h underflow the fp32 sigmoid to 0, so w1 / h1 is 0/0 and the row's
    CIoU is NaN in the reference; lbox, the loss and the four box logits of that cell are NaN, nothing else."""
    tg = [grid_target(0, 1, 4.5, 4.5, 2.0, 1.5, 32, 32), grid_target(0, 0, 17.3, 9.8, 1.7, 1.1, 32, 32)]
    c = make("ciou_nan", 1, 512, 512, 2, 2, TIE_ANCH, tg, 525)
    c["preds"][0][0, 2:4, 4, 4] = -200.0                              # target 0's centre row: image 0, anchor 0, cell (4, 4)

    def zero_box(case):
        r = _row(case, 0, 0, 0)
        with np.errstate(over="ignore"):
            s = f32(1) / (f32(1) + np.exp(-case["preds"][0][0, 2:4, 4, 4]))
        return r["gj"] == 4 and r["gi"] == 4 and not s.any()
    c["checks"].append(("zero-size predicted box", zero_box))
    return c


def case_big640():
    rs = np.random.RandomState(525)
    return make("big640", 2, 640, 640, 3, 80, COCO_ANCHORS, random_targets(rs, 25, 2, 80), 526, golden=False)


def case_wide():
    rs = np.random.RandomState(527)
    return make("wide352x640", 4, 352, 640, 2, 150, COCO_ANCHORS[:8], random_targets(rs, 30, 4, 150), 528, golden=False)


def case_a8_3000():
    rs = np.random.RandomState(529)
    anchors = list(np.round(rs.uniform(8, 200, 32), 2))
    return make("a8_nt3000", 16, 352, 352, 8, 20, anchors, random_targets(rs, 3000, 16, 20), 530, golden=False)


def all_cases():
    return ([case_ratio(), case_offsets(), case_borders(), case_empty(), case_tiny32(), case_reject_level1(), case_reject_all()]
            + [case_chunk(A, nt) for A, nt in ((1, 204), (1, 205), (5, 41), (1, 409), (2, 205))]
            + [case_same_cell(), case_saturated(), case_cls_tied(), case_a8_c150(), case_n64(), case_ciou_ties(), case_ciou_identical(), case_ciou_nan(),
               case_big640(), case_wide(), case_a8_3000()])


def check_sides(case):
    """Asserts that every input of the case sits on the side it was built for, and that every target is valid."""
    t = case["targets"]
    assert t.dtype == f32 and t.shape[1] == 6
    assert np.all((t[:, 0] >= 0) & (t[:, 0] < case["N"]) & (t[:, 0] == np.floor(t[:, 0]))), case["name"]
    assert np.all((t[:, 1] >= 0) & (t[:, 1] < case["C"]) & (t[:, 1] == np.floor(t[:, 1]))), case["name"]
    assert np.all((t[:, 2:] >= 0) & (t[:, 2:] <= 1)), case["name"]
    for lv, ti, a, want in case["sides"]:
        d = decide(case, lv)
        got = {"accept": bool(d["accept"][a, ti])}
        got.update({k: bool(d["flags"][i + 1, ti]) for i, k in enumerate("jklm")})
        for k, v in want.items():
            assert got[k] == v, (case["name"], lv, ti, a, k, got, float(d["ratio"][a, ti]))
    for lv, ti, o, a, want in case["ties"]:
        rel = row_relation(case, lv, ti, o, a)
        for k, v in want.items():
            if k == "tied":
                assert rel["tied"] == v, (case["name"], lv, ti, o, a, rel)
            elif k == "identical":
                assert rel["identical"] == v, (case["name"], rel)
            elif k == "iw_zero":
                assert rel["iw_raw"] == 0.0, (case["name"], rel)
            elif k == "iw_neg":
                assert rel["iw_raw"] < 0.0, (case["name"], rel)
            elif k == "ih_neg":
                assert rel["ih_raw"] < 0.0, (case["name"], rel)
    for what, fn in case["checks"]:
        assert fn(case), (case["name"], what)

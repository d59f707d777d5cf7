"""Host-side restatements of the choices k_post.cu makes from its arguments, and seeded inputs that land on chosen sides of them.

The NMS kernels pick a sort (by the candidate count), a suppression policy (dense scan or per-class kept lists) and, per IoU
test, an fp32 estimate or the exact fp64 comparison.  The results must not depend on the choice, so the tests build inputs for
each choice, assert on the host that every input sits on the side it was built for, and compare the kernel's rows and kept
indices bit for bit with oracle.post.  Everything here is numpy; nothing needs a GPU.
"""
import numpy as np

f32 = np.float32

NT = 256                  # threads per NMS CTA
NMS_CHUNK = 64            # candidates per suppression chunk
LIST_MIN_DET = 513        # kNmsListMinDet
LIST_CLASSES = 256        # kNmsListClasses
SMEM_CAP = 227 * 1024     # kSmemCap
MAX_CAND = 8192           # YFV2_NMS_MAX_CAND


def pow2_at_least(m, lo=64):
    p = lo
    while p < m:
        p <<= 1
    return p


def nms_smem_bytes(M, max_det):
    """k_post.cu nms_smem_bytes: shared memory of one NMS CTA (without the warp-per-cell staging of the fused kernel)."""
    MCp = pow2_at_least(M)
    b = MCp * 8 + M * 16 + ((M * 2 + 15) & ~15)
    b += max_det * 16 + ((max_det * 4 + 15) & ~15)
    b += 2 * NMS_CHUNK * 16 + 2 * NMS_CHUNK * 4 + NMS_CHUNK * 8 + NMS_CHUNK + 2 * NMS_CHUNK * 2 + 32
    return b


def largest_cap(M, extra=0):
    """The largest max_det (<= 4096) whose NMS state (plus `extra` bytes) fits in shared memory for M rows per image."""
    d = 4096
    while nms_smem_bytes(M, d) + extra > SMEM_CAP:
        d -= 1
    return d


def lists_fit(M, max_det):
    """The per-class kept lists live in the padding tail of the sort keys (entries [M, MCp))."""
    return 8 * M + 4 * max_det + 2 * LIST_CLASSES <= 8 * pow2_at_least(M) and max_det * 16 >= LIST_CLASSES * 4


def iou_mid(thr):
    """Rounding boundary between the two floats that bracket thr: fl32(q) > thr  <=>  q > mid (>= when tie_up)."""
    f0 = f32(thr)
    if float(f0) > thr:
        f0 = np.nextafter(f0, f32(-np.inf))
    f1 = np.nextafter(f0, f32(np.inf))
    return (float(f0) + float(f1)) * 0.5, bool((f1.view(np.uint32) & 1) == 0)


def candidates(x, conf_thres):
    """The reference's candidate filter on one image x [M, 5+C] (utils/utils.py:254-268): returns (xyxy boxes, conf, class, row)."""
    x = np.asarray(x, dtype=f32)
    ct = f32(conf_thres)
    rows = np.nonzero(x[:, 4] > ct)[0]
    y = x[rows]
    prob = y[:, 5:] * y[:, 4:5]
    j = prob.argmax(1) if len(rows) else np.zeros(0, np.int64)
    conf = prob[np.arange(len(rows)), j]
    m = conf > ct
    y, j, conf, rows = y[m], j[m], conf[m], rows[m]
    hw, hh = y[:, 2] * f32(0.5), y[:, 3] * f32(0.5)
    box = np.stack((y[:, 0] - hw, y[:, 1] - hh, y[:, 0] + hw, y[:, 1] + hh), 1).astype(f32)
    return box, conf, j, rows


def by_class(x, conf_thres, iou_thres, max_det, max_wh, lists_always=False):
    """sort_and_suppress's choice of the per-class kept lists for one image, restated: the lists fit, every candidate box lies
    inside (-max_wh/2, max_wh/2), the threshold's rounding boundary is positive, max_wh > 0, at most 256 classes, a cap of at least
    kNmsListMinDet (any cap with YFV2_NMS_LISTS set) and no class holding more than half of the candidates."""
    C = x.shape[1] - 5
    box, _, cls, _ = candidates(x, conf_thres)
    lim = f32(0.5) * f32(max_wh)
    inside = bool(np.all(np.abs(box) < lim))
    hist = np.bincount(cls, minlength=1)
    no_majority = not np.any(2 * hist > len(cls))
    return (lists_fit(x.shape[0], max_det) and inside and iou_mid(iou_thres)[0] > 0.0 and max_wh > 0 and C <= LIST_CLASSES
            and max_det >= (0 if lists_always else LIST_MIN_DET) and no_majority)


def sort_size(cnt):
    """n2: the bitonic network sorts the candidate keys padded to a power of two of at least 64."""
    return pow2_at_least(cnt)


# ------------------------------------------------------------------------------------------------------------------------------
# inputs for yfv2_nms: [N, M, 5+C] rows (cx, cy, w, h, obj, class scores)

def rows_from_boxes(boxes, conf, cls, C):
    """Decoded rows whose candidate boxes are exactly `boxes` (xyxy), with obj = 1 and class score `conf` on class `cls`."""
    boxes = np.asarray(boxes, np.float64)
    n = boxes.shape[0]
    d = np.zeros((n, 5 + C), f32)
    d[:, 0] = (boxes[:, 0] + boxes[:, 2]) * 0.5
    d[:, 1] = (boxes[:, 1] + boxes[:, 3]) * 0.5
    d[:, 2] = boxes[:, 2] - boxes[:, 0]
    d[:, 3] = boxes[:, 3] - boxes[:, 1]
    d[:, 4] = 1.0
    d[np.arange(n), 5 + np.asarray(cls)] = np.asarray(conf, f32)
    return d


def random_dets(seed, n, m, classes=80, side=640.0, size=None, n_pass=None, majority=None, half=False):
    """Random decoded rows.  n_pass: exactly this many rows pass conf_thres <= 1e-3 (the others have obj = 0).  majority: this
    class wins the arg-max on 60 % of the passing rows; half: class 0 wins on exactly half of them (the tie of the no-majority
    test).  size: box sides in [1, size] instead of up to side/3."""
    rs = np.random.RandomState(seed)
    d = np.zeros((n, m, 5 + classes), f32)
    d[..., 0:2] = (rs.rand(n, m, 2) * side).astype(f32)
    hi = side / 3 if size is None else size
    d[..., 2:4] = (1.0 + rs.rand(n, m, 2) * (hi - 1.0)).astype(f32)
    d[..., 4] = (0.05 + 0.95 * rs.rand(n, m)).astype(f32)
    c = rs.rand(n, m, classes).astype(f32)
    c = c * c
    c = c * c
    d[..., 5:] = c * f32(0.5)
    k = m if n_pass is None else n_pass
    for i in range(n):
        live = np.sort(rs.permutation(m)[:k])
        dead = np.setdiff1d(np.arange(m), live)
        d[i, dead, 4] = 0.0
        if majority is not None or half:
            nwin = (k * 3) // 5 + 1 if majority is not None else k // 2
            win = live[rs.permutation(k)[:nwin]]
            d[i, win, 5 + (majority if majority is not None else 0)] = f32(0.75) + f32(0.25) * rs.rand(nwin).astype(f32)
            if half:                      # every other passing row must not pick class 0
                rest = np.setdiff1d(live, win)
                d[i, rest, 5] = 0.0
    return d


def near_mid_pairs(thr, n_each, seed, rel=1e-6, side=1000, min_side=40):
    """Integer-corner box pairs (a, b) with sides below `side` whose exact IoU lies within `rel` (relative) of the rounding
    boundary `mid` of thr, n_each on each side of it.  The fp32 estimate of iou_fast cannot decide these; iou_gt's fp64 test must.
    At most two of them have an IoU of exactly thr (as a decimal fraction: 2/5 lies above the boundary of 0.4, since fl32(0.4) >
    0.4); the others are drawn past those.  Returns (a [k,4], b [k,4], q_above_mid [k] bool, rel_dist [k])."""
    from fractions import Fraction
    mid, _ = iou_mid(thr)
    fr = Fraction(str(thr))
    rs = np.random.RandomState(seed)
    got = {True: [], False: []}
    n_exact = 0
    for _ in range(200):
        if min(len(got[True]), len(got[False])) >= n_each:
            break
        K = 4000
        wa, ha = rs.randint(min_side, side, K), rs.randint(min_side, side, K)
        r = np.sqrt(mid)                                         # inter / area(a) >= mid leaves room for b
        iw = np.maximum(1, (rs.uniform(r, 1.0, K) * wa).astype(np.int64))
        ih = np.maximum(1, (rs.uniform(r, 1.0, K) * ha).astype(np.int64))
        inter = iw * ih
        lo = inter / (mid * (1 + rel)) - wa * ha + inter         # range of wb*hb
        hi = inter / (mid * (1 - rel)) - wa * ha + inter
        for k in np.nonzero(np.floor(hi) >= np.maximum(np.ceil(lo), 1))[0]:
            for nb in range(max(1, int(np.ceil(lo[k]))), int(np.floor(hi[k])) + 1):
                wbs = np.arange(max(int(iw[k]), -(-nb // (side - 1))), min(side - 1, nb // int(ih[k])) + 1)
                wbs = wbs[nb % wbs == 0] if len(wbs) else wbs
                if not len(wbs):
                    continue
                wb = int(wbs[rs.randint(len(wbs))])
                hb = nb // wb
                u = int(wa[k] * ha[k]) + nb - int(inter[k])
                d = float(inter[k]) - mid * u                    # exact: mid has 25 significant bits, u < 2^21
                exact = int(inter[k]) * fr.denominator == fr.numerator * u
                side_ = d > 0
                if d == 0.0 or (exact and n_exact >= 2) or len(got[side_]) >= n_each:
                    continue
                x0, y0 = int(wa[k] - iw[k]), int(ha[k] - ih[k])
                got[side_].append(((0, 0, int(wa[k]), int(ha[k])), (x0, y0, x0 + wb, y0 + hb), side_, abs(d / (mid * u))))
                n_exact += exact
    assert min(len(got[True]), len(got[False])) >= n_each, "no pairs found"
    allp = got[True] + got[False]
    return (np.array([p[0] for p in allp], np.float64), np.array([p[1] for p in allp], np.float64),
            np.array([p[2] for p in allp]), np.array([p[3] for p in allp]))


def fp32_estimate_disagrees(a, b, thr):
    """Pairs for which the fp32 pre-test of iou_fast WITHOUT its 1e-6 guard band (inter against fl(fl(mid) * u) alone) answers
    differently from the exact test: the pairs that need the fp64 path."""
    mid, tie_up = iou_mid(thr)
    aa = ((a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1])).astype(f32)
    ab = ((b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])).astype(f32)
    w = np.maximum(0, np.minimum(a[:, 2], b[:, 2]) - np.maximum(a[:, 0], b[:, 0]))
    h = np.maximum(0, np.minimum(a[:, 3], b[:, 3]) - np.maximum(a[:, 1], b[:, 1]))
    inter = (w * h).astype(f32)
    u = (aa + ab - inter).astype(f32)
    tq = (f32(mid) * u).astype(f32)
    exact = inter.astype(np.float64) >= mid * u.astype(np.float64) if tie_up else inter.astype(np.float64) > mid * u.astype(np.float64)
    est = np.where(inter > tq, True, np.where(inter < tq, False, exact))
    return est != exact


def pair_image(a, b, layout, C=80):
    """One image holding pair p in class p (pairs never interact: the classes sit max_wh apart).  layout "adjacent": the two
    boxes of a pair are neighbours in score order (tested inside one chunk); "split": every first box outranks every second one, so
    the second boxes meet their partners in the kept list (the chunk-against-kept phase)."""
    k = a.shape[0]
    assert k <= C
    p = np.arange(k)
    if layout == "adjacent":
        ca, cb = f32(0.9) - f32(0.002) * p, f32(0.899) - f32(0.002) * p
    else:
        ca, cb = f32(0.9) - f32(0.001) * p, f32(0.5) - f32(0.001) * p
    d = np.concatenate((rows_from_boxes(a, ca, p, C), rows_from_boxes(b, cb, p, C)), 0)
    perm = np.random.RandomState(k).permutation(2 * k)
    return d[perm]


def degenerate_image(seed, C=4):
    """Raw rows with zero-area boxes, negative widths and heights, identical boxes and ordinary ones, few classes."""
    rs = np.random.RandomState(seed)
    m = 96
    d = np.zeros((m, 5 + C), f32)
    d[:, 0:2] = rs.randint(0, 64, (m, 2)).astype(f32)
    d[:, 2:4] = rs.randint(1, 24, (m, 2)).astype(f32)
    d[0:12, 2] = 0.0                                # zero width
    d[12:20, 3] = 0.0                               # zero height
    d[20:24, 2:4] = 0.0                             # points
    d[24:36, 2] *= -1                               # negative width
    d[36:44, 2:4] *= -1                             # negative width and height (positive area)
    d[44:56] = d[56:68]                             # identical rows (boxes and scores)
    d[:, 4] = rs.choice([0.5, 0.75, 1.0], m).astype(f32)
    d[:, 5 + rs.randint(0, C, m)] = 0.0
    d[np.arange(m), 5 + rs.randint(0, C, m)] = rs.choice([0.25, 0.5, 0.625, 1.0], m).astype(f32)
    return d


def tie_image(seed, m=1815, C=80, side=640.0):
    """Scores with exact ties straddling sorted positions 64 (a chunk boundary) and 300 (the reference's cap).  Boxes are small
    and mostly apart, so nearly every candidate is kept and the tied ones decide the output; inside each tied run, pairs of
    identical boxes of one class make the lower row the one kept (stable order)."""
    rs = np.random.RandomState(seed)
    d = np.zeros((m, 5 + C), f32)
    d[:, 0:2] = (rs.rand(m, 2) * side).astype(f32)
    d[:, 2:4] = (2.0 + rs.rand(m, 2) * 6.0).astype(f32)
    d[:, 4] = 1.0
    conf = np.linspace(0.95, 0.05, m).astype(f32)
    conf[50:80] = conf[50]
    conf[285:320] = conf[285]
    order = rs.permutation(m)                       # row order differs from score order
    cls = rs.randint(0, C, m)
    for lo, hi in ((50, 80), (285, 320)):
        for q in range(lo, hi - 1, 3):              # rows of sorted positions q and q+1 share box and class
            r0, r1 = order[q], order[q + 1]
            d[r1, 0:4] = d[r0, 0:4]
            cls[r1] = cls[r0]
    d[order, 5 + cls[order]] = conf
    return d


def _corners(r, off):
    hw, hh = r[:, 2] * f32(0.5), r[:, 3] * f32(0.5)
    b = np.stack((r[:, 0] - hw, r[:, 1] - hh, r[:, 0] + hw, r[:, 1] + hh), 1).astype(f32)
    return (b + f32(off)).astype(f32)


def iou_parts(ra, rb, off=0.0):
    """(inter, union) of the candidate boxes of rows ra, rb [k, 5+] after the class offset `off`, in the fp32 arithmetic of
    torchvision's kernel (and of k_post.cu)."""
    A, B = _corners(ra, off), _corners(rb, off)
    aa = ((A[:, 2] - A[:, 0]) * (A[:, 3] - A[:, 1])).astype(f32)
    ab = ((B[:, 2] - B[:, 0]) * (B[:, 3] - B[:, 1])).astype(f32)
    w = np.maximum(f32(0), np.minimum(A[:, 2], B[:, 2]) - np.maximum(A[:, 0], B[:, 0]))
    h = np.maximum(f32(0), np.minimum(A[:, 3], B[:, 3]) - np.maximum(A[:, 1], B[:, 1]))
    inter = (w * h).astype(f32)
    return inter, ((aa + ab).astype(f32) - inter).astype(f32)


def estimate_disagrees(inter, u, thr):
    """Whether the fp32 estimate inter vs fl(fl(mid) * u), WITHOUT the 1e-6 guard band of iou_fast, answers differently from the
    exact test (fl32(inter / u) > thr, i.e. inter > mid * u in exact arithmetic)."""
    mid, tie_up = iou_mid(thr)
    rhs = mid * u.astype(np.float64)                             # exact: 25 x 24 significant bits
    exact = inter.astype(np.float64) >= rhs if tie_up else inter.astype(np.float64) > rhs
    tq = (f32(mid) * u).astype(f32)
    est = np.where(inter > tq, True, np.where(inter < tq, False, exact))
    return est != exact


def zone_heights(thr, n, seed):
    """Heights (ha, hb) of n box pairs a = (x, 0, x+1, ha), b = (x, 0, x+1, hb) (b inside a, IoU about hb / ha) whose fp32 IoU
    lies between the rounding boundary `mid` of thr and the fp32 product fl(fl(mid) * union): the pairs an fp32 estimate of the
    boundary alone misjudges, so only the exact fp64 test keeps the kernel right.  There are none for some thresholds (0.45: the
    gap between fl32(0.45) and the boundary is below half an ulp of the product); at most n.  Returns (ha, hb, suppressed)."""
    mid, tie_up = iou_mid(thr)
    rs = np.random.RandomState(seed)
    ha = rs.uniform(96 / mid, 128 / mid, 200000).astype(f32)       # IoU in the top of a binade: the estimate is coarsest there
    hb0 = (ha.astype(np.float64) * mid).astype(f32)
    for k in range(-3, 4):
        hb = (hb0.view(np.int32) + np.int32(k)).view(f32)
        ra = np.stack((np.full_like(ha, 0.5), ha * f32(0.5), np.ones_like(ha), ha), 1)
        rb = np.stack((np.full_like(hb, 0.5), hb * f32(0.5), np.ones_like(hb), hb), 1)
        inter, u = iou_parts(ra, rb)
        dis = estimate_disagrees(inter, u, thr)
        if k == -3:
            hits_a, hits_b, hits_u, hits_i = ha[dis], hb[dis], u[dis], inter[dis]
        else:
            hits_a, hits_b = np.concatenate((hits_a, ha[dis])), np.concatenate((hits_b, hb[dis]))
            hits_u, hits_i = np.concatenate((hits_u, u[dis])), np.concatenate((hits_i, inter[dis]))
    pick = rs.permutation(len(hits_a))[:n]
    rhs = mid * hits_u[pick].astype(np.float64)                   # exact: 25 x 24 significant bits
    sup = hits_i[pick].astype(np.float64) >= rhs if tie_up else hits_i[pick].astype(np.float64) > rhs
    return hits_a[pick], hits_b[pick], sup


def zone_image(thr, n, seed, layout, m=160, C=80):
    """One image with n zone pairs (zone_heights) side by side in class 0, and 64 - n small far-apart class-1 boxes that are all
    kept.  layout "adjacent": each pair is consecutive in score order (one chunk); "split": all first boxes, then the class-1
    boxes, then the second boxes (chunk 1 meets its partners among the 64 kept boxes of chunk 0).  Returns (rows [m, 5+C],
    suppressed [n])."""
    ha, hb, sup = zone_heights(thr, n, seed)
    x = np.arange(n, dtype=np.float64) * 2
    a = np.stack((x, np.zeros(n), x + 1, ha), 1)
    b = np.stack((x, np.zeros(n), x + 1, hb), 1)
    nf = 64 - n
    fx = 1000 + (np.arange(nf) % 8) * 20.0
    fy = 1000 + (np.arange(nf) // 8) * 20.0
    fil = np.stack((fx, fy, fx + 2, fy + 2), 1)
    p = np.arange(n)
    if layout == "adjacent":
        ca, cb, cf = f32(0.9) - f32(0.004) * p, f32(0.898) - f32(0.004) * p, f32(0.5) - f32(0.001) * np.arange(nf)
    else:
        ca, cb, cf = f32(0.9) - f32(0.001) * p, f32(0.3) - f32(0.001) * p, f32(0.6) - f32(0.001) * np.arange(nf)
    d = np.zeros((m, 5 + C), f32)
    d[:2 * n + nf] = np.concatenate((rows_from_boxes(a, ca, np.zeros(n, int), C), rows_from_boxes(b, cb, np.zeros(n, int), C),
                                     rows_from_boxes(fil, cf, np.ones(nf, int), C)), 0)
    return d[np.random.RandomState(seed + 1).permutation(m)], sup

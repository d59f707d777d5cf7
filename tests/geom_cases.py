"""Seeded cases of the geometric augmentation (yfv2_aug_geometric, utils.device_aug.geometric_targets): batches, targets and
per-image draws.  tests/golden/make_golden_geom.py freezes cv2's bytes and YOLOv5's labels for them, together with each case's
draws (the matrices come from cos, sin and tan, so the tests read them back from the golden file instead of recomputing them)."""
import math
import random

import numpy as np

# name, N, H, W, seed, how the draws are made: ("hyp", {...}) through draw_geometric, or ("explicit", fn(N, H, W) -> draws)
IDENT = np.eye(3)


def _draw(mosaic=0, src=(0, 0, 0, 0), xc=0, yc=0, M=IDENT, perspective=0, flip=0, s=1.0):
    return dict(mosaic=bool(mosaic), src=list(src), xc=xc, yc=yc, M=np.asarray(M, np.float64), perspective=bool(perspective),
                flip=bool(flip), s=s)


def rot(angle, scale, cw, ch, W, H):
    """T @ R @ C of random_perspective with the given angle and scale, the canvas centre to the output centre."""
    a = angle * (math.pi / 180)
    al, be = math.cos(a) * scale, math.sin(a) * scale
    C = np.array([[1, 0, -cw / 2], [0, 1, -ch / 2], [0, 0, 1]], np.float64)
    R = np.array([[al, be, 0], [-be, al, 0], [0, 0, 1]], np.float64)
    T = np.array([[1, 0, W / 2], [0, 1, H / 2], [0, 0, 1]], np.float64)
    return T @ R @ C


def _rotations(angle, scale, mosaic=False):
    def fn(N, H, W):
        cw, ch = (2 * W, 2 * H) if mosaic else (W, H)
        return [_draw(mosaic, [i, (i + 1) % N, (i + 2) % N, (i + 3) % N], W, H, rot(angle, scale, cw, ch, W, H), s=scale)
                for i in range(N)]
    return fn


def _ends(N, H, W):
    """xc, yc at both ends of their range: two quadrants clipped away, the others partly 114."""
    out = []
    for i in range(N):
        lo = i % 2 == 0
        xc, yc = (W // 2, H // 2) if lo else (2 * W - W // 2, 2 * H - H // 2)
        out.append(_draw(1, [i, (i + 1) % N, (i + 2) % N, (i + 3) % N], xc, yc, rot(3.0 * i, 1.0, 2 * W, 2 * H, W, H)))
    return out


def _repeated(N, H, W):
    return [_draw(1, [0, 0, 1, 0], W - 5, H + 7, rot(0, 1.0, 2 * W, 2 * H, W, H)),
            _draw(1, [2, 2, 2, 1], W + 9, H - 3, rot(10, 0.8, 2 * W, 2 * H, W, H), flip=1, s=0.8),
            _draw(1, [1, 1, 1, 1], W, H, rot(-5, 1.2, 2 * W, 2 * H, W, H), s=1.2)]


def _ties(N, H, W):
    """Exact-half fixed-point coordinates: (m1 y + m2) 1024 = k + 1/2 for the affine warp, ((m1 y + m2) + m0 x) 32 = k + 1/2 for
    the perspective one (M's inverse is exact: unit diagonal, so m2 = -M[0, 2])."""
    return [_draw(0, [0] * 4, M=[[1, 0, -3 / 2048], [0, 1, 5 / 2048], [0, 0, 1]]),
            _draw(0, [1] * 4, M=[[1, 0, 1 / 2048], [0, 1, -7 / 2048], [0, 0, 1]], flip=1),
            _draw(0, [0] * 4, M=[[1, 0, -3 / 64], [0, 1, 5 / 64], [0, 0, 1]], perspective=1),
            _draw(0, [1] * 4, M=[[1, 0, 1 / 64], [0, 1, -1 / 64], [0, 0, 1]], perspective=1, flip=1)]


def _fma(N, H, W):
    """Row 3, column 0 computes fl(fl(1/3) * 3) + m2 = 1 + m2 (the product rounds to 1), with (1 + m2) * 1024 = 15.5 (affine:
    rounded half to even to 16, so X = (16 + 16) >> 5 = 1) or (1 + m2) * 32 = 1.5 (perspective: X = 2).  A fused multiply-add
    keeps the product's 2^-54 shortfall and rounds to 15 (X = 0) or 1."""
    return [_draw(0, [0] * 4, M=[[1, -1 / 3, 1 - 15.5 / 1024], [0, 1, 0], [0, 0, 1]]),
            _draw(0, [1] * 4, M=[[1, -1 / 3, 1 - 1.5 / 32], [0, 1, 0], [0, 0, 1]], perspective=1)]


def _flip(flip):
    def fn(N, H, W):
        d = [dict(x) for x in draw_hyp(N, H, W, 11, dict(mosaic=0.5, degrees=10, shear=3))]
        for x in d:
            x["flip"] = bool(flip)
        return d
    return fn


def draw_hyp(N, H, W, seed, hyp):
    import utils.device_aug as da
    return da.draw_geometric(N, H, W, random.Random(seed), **hyp)


MIXED = dict(mosaic=0.5, degrees=10, translate=0.1, scale=0.5, shear=5, perspective=0.0, fliplr=0.5)
CASES = [
    ("identity", 2, 48, 64, 1, ("explicit", lambda N, H, W: [_draw(0, [i] * 4) for i in range(N)])),
    ("affine", 3, 96, 96, 2, ("hyp", dict(mosaic=0, degrees=10, shear=5))),
    ("perspective", 3, 96, 96, 3, ("hyp", dict(mosaic=0, degrees=10, shear=5, perspective=0.001))),
    ("mosaic_ends", 4, 64, 64, 4, ("explicit", _ends)),
    ("mosaic_n1", 1, 64, 64, 5, ("hyp", dict(mosaic=1, degrees=5, perspective=0.0005))),
    ("repeated", 3, 64, 64, 6, ("explicit", _repeated)),
    ("rot90", 2, 64, 64, 7, ("explicit", _rotations(90, 1.0))),
    ("rot45", 2, 64, 64, 8, ("explicit", _rotations(45, 1.0, mosaic=True))),
    ("scale05", 2, 64, 64, 9, ("explicit", _rotations(0, 0.5))),
    ("scale15", 2, 64, 64, 10, ("explicit", _rotations(0, 1.5, mosaic=True))),
    ("flip_on", 4, 64, 64, 11, ("explicit", _flip(1))),
    ("flip_off", 4, 64, 64, 11, ("explicit", _flip(0))),
    ("nonsquare", 4, 192, 320, 12, ("hyp", dict(mosaic=0.75, degrees=10, shear=3, perspective=0.0005))),
    ("tiny", 4, 32, 32, 13, ("hyp", MIXED)),
    ("ties", 4, 64, 64, 14, ("explicit", _ties)),
    ("fma", 2, 16, 16, 17, ("explicit", _fma)),
    ("defaults", 8, 96, 96, 15, ("hyp", {})),
    ("jpeg", 2, 96, 96, 16, ("hyp", dict(mosaic=1, degrees=10, shear=5, perspective=0.001))),
]
JPEGS = ("000004.jpg", "000139.jpg")


def images(name, N, H, W, seed, jpeg=None):
    """The case's planar [N, 3, H, W] uint8 batch: smooth gradients with noise (so every sample's four taps differ), or for "jpeg"
    the bundled images as cv2.imread + cv2.resize to W x H gave them (jpeg: [N, H, W, 3] from the golden file)."""
    if name == "jpeg":
        return np.ascontiguousarray(np.asarray(jpeg).transpose(0, 3, 1, 2))
    rs = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:H, 0:W]
    base = np.stack([(xx * 255 // max(W - 1, 1)), (yy * 255 // max(H - 1, 1)), ((xx + yy) * 7) % 256])[None]
    noise = rs.randint(-40, 41, (N, 3, H, W))
    return np.clip(base + noise + rs.randint(-60, 61, (N, 3, 1, 1)), 0, 255).astype(np.uint8)


def targets(N, seed):
    """Rows (image, class, cx, cy, w, h) float32: 1 to 5 boxes per image, some near the edges."""
    rs = np.random.RandomState(1000 + seed)
    rows = []
    for n in range(N):
        for _ in range(rs.randint(1, 6)):
            w, h = rs.uniform(0.05, 0.6), rs.uniform(0.05, 0.6)
            rows.append([n, rs.randint(0, 80), rs.uniform(0.02, 0.98), rs.uniform(0.02, 0.98), w, h])
    return np.array(rows, np.float32)


def draws(case):
    name, N, H, W, seed, (kind, arg) = case
    return draw_hyp(N, H, W, seed, arg) if kind == "hyp" else arg(N, H, W)


META_KEYS = ("mosaic", "src0", "src1", "src2", "src3", "xc", "yc", "flip", "perspective")


def pack(ds):
    """draws -> (M [N, 3, 3] float64, meta [N, 9] int64, s [N] float64), what the golden file stores."""
    M = np.stack([np.asarray(d["M"], np.float64) for d in ds])
    meta = np.array([[int(d["mosaic"])] + [int(v) for v in d["src"]] + [d["xc"], d["yc"], int(d["flip"]), int(d["perspective"])]
                     for d in ds], np.int64)
    return M, meta, np.array([d["s"] for d in ds], np.float64)


def unpack(M, meta, s):
    return [dict(mosaic=bool(r[0]), src=[int(v) for v in r[1:5]], xc=int(r[5]), yc=int(r[6]), flip=bool(r[7]),
                 perspective=bool(r[8]), M=M[i], s=float(s[i])) for i, r in enumerate(meta)]

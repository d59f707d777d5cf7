"""Seeded inputs of tests/golden/aug_blur_cases.npz (tests/golden/make_golden_aug_blur.py) and the tests that read it."""
import numpy as np

import aug_blur_oracle as bo

# taps: a dense sweep of angles for both degrees (digest), full arrays at a few, and the special angles
SWEEP = np.linspace(-360.0, 360.0, 28801)                    # 0.025 degree steps
FULL_ANGLES = (-300.5, -17.25, 33.3, 128.0, 271.9)
SPECIAL_ANGLES = (0.0, 45.0, -45.0, 90.0, -90.0, 180.0, -180.0, 360.0, -360.0)


def fixed_terms(degree, angle):
    """warpAffine's cvRound'ed fixed-point terms (row terms x0, y0 per row, column terms per column) and the 1/32-pixel source
    coordinates X, Y: where the 1/1024 and 1/32 rounding edges of the kernel lie."""
    im = bo.invert_affine(bo.rotation_matrix(degree, angle))
    terms = [round(float(im[1] * y + im[2]) * 1024) for y in range(degree)]
    terms += [round(float(im[4] * y + im[5]) * 1024) for y in range(degree)]
    terms += [round(im[0] * x * 1024) for x in range(degree)] + [round(im[3] * x * 1024) for x in range(degree)]
    X, Y = bo.warp_coords(degree, angle)
    return terms, np.concatenate([X.ravel(), Y.ravel()]).tolist()


def edge_pair(degree, a0, a1, which):
    """Bisects [a0, a1] (whose terms (which 0) or coordinates (which 1) differ) down to two adjacent doubles that differ."""
    f = lambda a: fixed_terms(degree, a)[which]                          # noqa: E731
    lo, hi = a0, a1
    flo = f(lo)
    assert flo != f(hi)
    while np.nextafter(lo, hi) != hi:
        mid = lo + (hi - lo) / 2
        if mid in (lo, hi):
            break
        if f(mid) == flo:
            lo = mid
        else:
            hi = mid
    return lo, hi


def find_edges(degree, which, count, seed):
    """count pairs of adjacent angles across which a 1/1024 term (which 0) or a 1/32 coordinate (which 1) changes."""
    rs = np.random.RandomState(seed)
    out = []
    while len(out) < count:
        a0 = rs.uniform(-360, 360)
        a1 = a0 + 0.5
        if fixed_terms(degree, a0)[which] != fixed_terms(degree, a1)[which]:
            out.append(edge_pair(degree, a0, a1, which))
    return out


# filter2D + normalize: (name, (seed, h, w), degree, angle); widths 1..64 and 352, a row, a column, 2 x 2
FILTER_CASES = [("w%d" % w, (200 + w, 1 + (7 * w) % 13, w), 2 + w % 2, -350.0 + 11.3 * w) for w in range(1, 65)]
FILTER_CASES += [("352_d2", (300, 352, 352), 2, 61.7), ("352_d3", (301, 352, 352), 3, -143.2),
                 ("row_d3", (302, 1, 45), 3, 17.0), ("col_d2", (303, 16, 1), 2, -77.0), ("col_d3", (304, 45, 1), 3, 200.0),
                 ("2x2_d2", (305, 2, 2), 2, 33.0), ("2x2_d3", (306, 2, 2), 3, 133.0), ("1x1_d3", (307, 1, 1), 3, 10.0)]


def image(seed, h, w):
    return np.random.RandomState(seed).randint(0, 256, (h, w, 3)).astype(np.uint8)


def constant_image(h=9, w=14, v=77):
    return np.full((h, w, 3), v, np.uint8)


def striped_image(h=12, w=20):
    """Rows alternating 100 and 101: degree 2 at angle 0 averages (y - 1, x - 1) and (y, x), 100.5 in every pixel, which
    rounds to 100 (half to even), so the blurred image is constant."""
    img = np.empty((h, w, 3), np.uint8)
    img[0::2], img[1::2] = 100, 101
    return img


# seeded motion_blur alone and the whole chain: per seed a batch of N 352 x 352 images
BLUR_SEEDS = (0, 3, 11)
CHAIN_SEEDS = (0, 5, 9)
SEEDED_N = 6


def seeded_batch(seed):
    return [image(500 + 10 * seed + i, 352, 352) for i in range(SEEDED_N)]

"""Seeded frames and warp matrices for the goldens of tests/golden/make_golden_warp.py (cv2.cvtColor, cv2.warpAffine /
cv2.warpPerspective INTER_LINEAR, crop, cv2.resize INTER_LINEAR) and the tests.

A case is a dict: the inner frame (layout, seed, (fh, fw), `inner`: a window of it the warp addresses, or None), the matrix
(`M`: 2x3 or 3x3 float64 as cv2 takes it), `inverse` (cv2.WARP_INVERSE_MAP), `dsize` (width, height), the window of the warped
image (`view`, None for all of it) and the resize target (W, H).  Matrices with a trigonometric part are stored in the golden
file as `<name>_M` (tests read them from there, so the cases do not depend on the platform's cos and sin); the others are exact
binary fractions.  INV_MATRICES builds the 3x3 matrices whose cv2.invert the golden file pins, from integers and powers of two
only."""
import numpy as np

import bayer_cases as bc
import remap_cases as rc

LAYOUTS = rc.LAYOUTS
CODES = rc.CODES
YUV420 = rc.YUV420
FULL_BYTES = 4 * 1024                            # outputs up to this size are stored whole, larger ones as SHA-256


def rotation(cx, cy, deg, scale=1.0):
    """cv2.getRotationMatrix2D((cx, cy), deg, scale)."""
    a = np.deg2rad(deg)
    al, be = scale * np.cos(a), scale * np.sin(a)
    return np.array([[al, be, (1 - al) * cx - be * cy], [-be, al, be * cx + (1 - al) * cy]], np.float64)


def quad_homography(w, h, off):
    """The 3x3 matrix taking the corners of a w x h image to the corners moved by off (4 x 2, fractions of w and h), solved in
    float64 as cv2.getPerspectiveTransform's linear system (any exact solver: the matrix is data, stored in the golden file)."""
    src = np.array([[0, 0], [w, 0], [w, h], [0, h]], np.float64)
    dst = src + np.asarray(off, np.float64) * [w, h]
    A, b = [], []
    for (x, y), (u, v) in zip(src, dst):
        A.append([x, y, 1, 0, 0, 0, -u * x, -u * y])
        A.append([0, 0, 0, x, y, 1, -v * x, -v * y])
        b += [u, v]
    return np.append(np.linalg.solve(np.array(A), np.array(b)), 1.0).reshape(3, 3)


def birdseye(w, h, dw, dh, horizon):
    """A destination -> source ground-plane rectification (use with inverse) of a w x h frame into dw x dh, whose W = 0 line is
    output row `horizon`: rows above it see the sky behind the camera, rows below the road."""
    return np.array([[w / dw, -0.35 * w / dh, 0.1 * w], [0.0, 0.2 * h / dh, 0.0], [0.0, 1.0 / dh, -horizon / dh]], np.float64)


ROT90 = {"ccw": lambda w, h: np.array([[0, 1, 0], [-1, 0, w - 1]], np.float64),
         "180": lambda w, h: np.array([[-1, 0, w - 1], [0, -1, h - 1]], np.float64),
         "cw": lambda w, h: np.array([[0, -1, h - 1], [1, 0, 0]], np.float64)}


def _case(name, layout, size, M, dsize, inverse=False, view=None, target=(64, 48), inner=None, rotate=None):
    return {"name": name, "layout": layout, "size": size, "M": np.asarray(M, np.float64), "dsize": dsize, "inverse": inverse,
            "view": view, "target": target, "inner": inner, "rotate": rotate}


def _cases():
    cases = []
    rs = np.random.RandomState(1900)
    for k, layout in enumerate(LAYOUTS):
        fh, fw = 76, 98
        cases.append(_case(layout + "_rot", layout, (fh, fw), rotation(49, 38, 17 + 11 * k, 0.9), (90, 70), inverse=bool(k % 2)))
        off = rs.uniform(-0.25, 0.25, (4, 2))
        cases.append(_case(layout + "_persp_window", layout, (fh, fw), quad_homography(fw, fh, off), (110, 84),
                           inverse=bool(k % 3 == 0), view=(5, 7, 80, 60), target=(352, 352)))
    cases += [
        _case("bayer_gr_ea_inner_window", "bayer_gr_ea", (76, 98), rotation(40, 30, -31, 1.1), (80, 60), inner=(3, 5, 90, 66)),
        _case("bayer_bg_inner_window_persp", "bayer_bg", (76, 98), quad_homography(55, 43, [[.1, 0], [-.1, .05], [0, 0], [.02, -.1]]),
              (61, 41), inner=(37, 21, 55, 43)),
        _case("bgr_inner_crop", "bgr", (120, 160), rotation(50, 35, 45), (100, 70), inner=(31, 17, 100, 70)),
        _case("nv12_inner_crop", "nv12", (120, 160), quad_homography(100, 70, [[0, .1], [0, -.1], [.1, 0], [-.1, 0]]), (100, 70),
              inner=(30, 18, 100, 70)),
        _case("bgr_rot90_ccw", "bgr", (47, 61), ROT90["ccw"](61, 47), (47, 61), target=(47, 61), rotate="ROTATE_90_COUNTERCLOCKWISE"),
        _case("bgr_rot180", "bgr", (47, 61), ROT90["180"](61, 47), (61, 47), target=(61, 47), rotate="ROTATE_180"),
        _case("bgr_rot90_cw", "bgr", (47, 61), ROT90["cw"](61, 47), (47, 61), target=(47, 61), rotate="ROTATE_90_CLOCKWISE"),
        _case("nv12_rot90_cw", "nv12", (48, 62), ROT90["cw"](62, 48), (48, 62), rotate="ROTATE_90_CLOCKWISE"),
        _case("bayer_rg_rot180", "bayer_rg", (41, 53), ROT90["180"](53, 41), (53, 41), rotate="ROTATE_180"),
        _case("bgr_rot_any", "bgr", (120, 160), rotation(80, 60, 33.3, 1.0), (160, 120), target=(128, 96)),
        _case("bgr_rot_neg_scaled", "bgr", (120, 160), rotation(10.5, 100.25, -127, 0.45), (200, 150), inverse=True),
        _case("gray_scale_up", "gray", (31, 41), [[2.5, 0, -3.25], [0, 3.125, 1.5]], (120, 100), target=(96, 80)),
        _case("bgr_scale_down", "bgr", (120, 160), [[0.3, 0, 2], [0, 0.27, -1]], (40, 30), target=(40, 30)),
        _case("bgr_shear", "bgr", (60, 80), [[1, 0.4, -10], [0.15, 1, 3]], (96, 72), target=(96, 72)),
        _case("yuyv_shear_inverse", "yuyv", (60, 80), [[1, -0.3, 12], [0.2, 0.9, -5]], (70, 50), inverse=True),
        _case("bgr_persp_random", "bgr", (120, 160), quad_homography(160, 120, rs.uniform(-.3, .3, (4, 2))), (150, 110)),
        _case("rgb_persp_random_inverse", "rgb", (120, 160), quad_homography(160, 120, rs.uniform(-.3, .3, (4, 2))), (150, 110),
              inverse=True),
        _case("bgr_birdseye", "bgr", (120, 160), birdseye(160, 120, 140, 120, 37.5), (140, 120), inverse=True, target=(96, 96)),
        _case("nv21_birdseye_forward", "nv21", (120, 160), birdseye(160, 120, 140, 120, 50.5), (140, 120), target=(70, 60)),
        # dst -> src with W = y / 32 - 2: exactly 0 on output row 64, where every pixel is source (0, 0) with code 0
        _case("bgr_horizon_row", "bgr", (90, 100), [[1, 0.5, 3], [0.25, 1, 2], [0, 0.03125, -2]], (100, 100), inverse=True,
              target=(100, 100)),
        _case("bayer_gb_horizon_row", "bayer_gb", (90, 100), [[-0.5, 1, 3], [0.25, -1, 80], [0, -0.03125, 2]], (100, 100),
              inverse=True),
        # 3x3 with last row [0, 0, 1]: warpPerspective's arithmetic (W = 32), half-way products at m2 = 1/64 and m5 = 3/64
        _case("bgr_persp_affine_row_ties", "bgr", (40, 50), [[1, 0, 1 / 64], [0, 1, 3 / 64], [0, 0, 1]], (50, 40), inverse=True,
              target=(50, 40)),
        _case("bgr_affine_ties", "bgr", (40, 50), [[1 + 1 / 2048, 0, 1 / 2048], [1 / 4096, 1 - 3 / 2048, 3 / 2048]], (50, 40),
              inverse=True, target=(50, 40)),
        _case("gray_persp_ties", "gray", (40, 50), [[0.5, 1 / 128, 1 / 64], [1 / 256, 0.5, 1 / 128], [0, 0, 0.5]], (60, 50),
              inverse=True),
        # the affine bound just inside: |(m1 y + m2) * 1024| = 2^30 - 1024 and |(m3 x) * 1024| = 2^30 - 2048 at the far side
        _case("bgr_affine_bound_row", "bgr", (20, 30), [[1, 0, 1048575.0], [0, 1, -1048575.0]], (8, 8), inverse=True,
              target=(8, 8)),
        _case("bgr_affine_bound_x", "bgr", (20, 30), [[1048574.0 / 1023, 0, 0], [-1048574.0 / 1023, 0, 5]], (1024, 3),
              inverse=True, target=(64, 3)),
        _case("bgr_px1x1", "bgr", (1, 1), rotation(0, 0, 30, 1.0), (5, 4), target=(4, 4)),
        _case("gray_px1x1", "gray", (1, 1), [[0.5, 0, -0.25], [0, 0.5, -0.25]], (3, 3)),
        _case("bayer_bg_px1x1", "bayer_bg", (1, 1), [[1, 0, 0], [0, 1, 0], [0, 0, 1]], (3, 3)),
        _case("bgr_out1x1", "bgr", (30, 40), rotation(20, 15, 10), (1, 1), target=(3, 3)),
        _case("bgr_win_far_corner", "bgr", (120, 160), rotation(80, 60, 21), (160, 120), view=(159, 119, 1, 1), target=(2, 5)),
        _case("nv21_win_odd", "nv21", (120, 160), quad_homography(160, 120, [[.1, .1], [-.1, .1], [-.1, -.1], [.1, -.1]]),
              (160, 120), view=(37, 21, 55, 43), target=(96, 96)),
        _case("bgr_output_larger", "bgr", (30, 40), rotation(20, 15, 5, 4.0), (300, 200), target=(160, 96)),
        _case("bgr_fullhd_rot", "bgr", (1080, 1920), rotation(960, 540, 7.5), (1920, 1080), target=(352, 352)),
        _case("nv12_fullhd_birdseye", "nv12", (1080, 1920), birdseye(1920, 1080, 1920, 1080, 300.5), (1920, 1080), inverse=True,
              target=(352, 352)),
        _case("bayer_bg_fullhd_persp", "bayer_bg", (1080, 1920),
              quad_homography(1920, 1080, [[.05, .02], [-.03, .04], [.02, -.05], [-.04, -.01]]), (1920, 1080), target=(352, 352)),
    ]
    for k, c in enumerate(cases):
        c["seed"] = 1900 + k
    return cases


CASES = _cases()
# cases whose matrix involves cos, sin or a solver: tests take M from the golden file
FROM_GOLDEN = {c["name"] for c in CASES if not np.array_equal(c["M"], np.round(c["M"] * 2 ** 20) / 2 ** 20)}


def case_matrix(c, golden=None):
    """The case's M as cv2 takes it: from the golden file when it has one, else the case's own exact values."""
    if golden is not None and c["name"] + "_M" in golden:
        return np.array(golden[c["name"] + "_M"], np.float64)
    return c["M"]


def frame(layout, seed, fh, fw):
    return rc.frame(layout, seed, fh, fw)


def case_frame(c):
    return frame(c["layout"], c["seed"], *c["size"])


def view_window(c):
    """(x0, y0, w, h) of the warped image the case resizes."""
    return c["view"] or (0, 0) + tuple(c["dsize"])


# encode cases: (case name, quality, sampling, region of the view's window or None): cv2.imencode of cv2's warped window
ENCODE_CASES = [("bgr_rot", 95, "420", None), ("nv12_persp_window", 90, "444", None), ("bayer_rg_rot", 75, "422", (10, 7, 61, 47)),
                ("bgr_birdseye", 85, "420", (3, 2, 100, 90)), ("gray_rot", 95, "420", None)]


def inv_matrices():
    """3x3 matrices for cv2.invert: well conditioned, ill-conditioned (a row almost the sum of the others), exactly singular, and
    spanning many binades, all built from integers and powers of two so that every platform builds the same values."""
    rs = np.random.RandomState(77)
    out = []
    for k in range(3000):
        m = np.ldexp(rs.randint(-2 ** 30, 2 ** 30, 9).astype(np.float64), rs.randint(-60, -10, 9))
        kind = k % 4
        if kind == 1:                              # ill-conditioned: row 2 = row 0 + row 1 + a tiny perturbation
            m[6:] = m[:3] + m[3:6] + np.ldexp(rs.randint(-1024, 1024, 3).astype(np.float64), -70)
        elif kind == 2:                            # exactly singular: row 2 = 2 * row 0 (exact in binary)
            if k % 8 == 2:
                m[6:] = 2 * m[:3]
        elif kind == 3:                            # entries of one magnitude: homographies as cameras give them
            m = np.ldexp(rs.randint(-2 ** 20, 2 ** 20, 9).astype(np.float64), -20)
            m[8] = 1.0
        out.append(m.reshape(3, 3))
    return np.array(out)

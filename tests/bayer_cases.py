"""Seeded raw Bayer frames for the goldens of tests/golden/make_golden_bayer.py (cv2.cvtColor(COLOR_Bayer??2BGR / _EA), then
cv2.resize INTER_LINEAR, a crop or cv2.imencode) and the tests.

A resize case is (name, layout, seed, (fh, fw), (H, W), window, form): a raw frame of noise or of a noisy gradient, drawn from
numpy's legacy RandomState (bit-stable across numpy versions); window (x0, y0, w, h) of the converted frame, None for all of it;
form None for a contiguous frame, ("pitch", SH, SW, y0, x0) for the frame as a view into a larger SH x SW surface.  The image cv2
resizes is cv2.cvtColor(raw, code)[y0:y0 + h, x0:x0 + w].  Every shape runs for all 8 layouts: every (fw mod 2, fh mod 2), 1-3
pixel sides, 1080p, pitched views, and windows that touch each edge, 1-pixel windows and odd offsets.

An encode case is a dict: the raw frame (layout, seed, fh, fw), the window of its conversion (or None), the region of the window
(or None) and cv2.imencode's quality and sampling."""
import numpy as np

import bayer_oracle as bo

LAYOUTS = bo.LAYOUTS
CODES = {"bayer_bg": "COLOR_BayerBG2BGR", "bayer_gb": "COLOR_BayerGB2BGR", "bayer_rg": "COLOR_BayerRG2BGR",
         "bayer_gr": "COLOR_BayerGR2BGR"}
CODES.update({k + "_ea": v + "_EA" for k, v in list(CODES.items())})
FULL_BYTES = 4 * 1024           # outputs up to this size are stored whole, larger ones as SHA-256

_SHAPES = [
    # name, (fh, fw), (H, W), window, form
    ("even_even", (480, 640), (352, 352), None, None),
    ("odd_even", (481, 640), (352, 352), None, None),
    ("even_odd", (480, 641), (96, 160), None, None),
    ("odd_odd", (481, 641), (29, 37), None, None),
    ("fullhd", (1080, 1920), (352, 352), None, None),
    ("fullhd_odd", (1081, 1921), (352, 352), None, None),
    ("px1x1", (1, 1), (4, 4), None, None),
    ("px1x5", (1, 5), (3, 7), None, None),
    ("px2x2", (2, 2), (5, 5), None, None),
    ("px2x9", (2, 9), (8, 12), None, None),
    ("px9x2", (9, 2), (12, 8), None, None),
    ("px3x3", (3, 3), (7, 9), None, None),
    ("px3x1000", (3, 1000), (24, 352), None, None),
    ("px1000x3", (1000, 3), (352, 24), None, None),
    ("px4x17", (4, 17), (30, 40), None, None),
    ("upscale", (12, 16), (96, 128), None, None),
    ("identity", (61, 83), (61, 83), None, None),
    ("pitched", (177, 333), (352, 352), None, ("pitch", 200, 400, 5, 7)),
    ("pitched_window", (121, 160), (64, 64), (37, 21, 55, 43), ("pitch", 130, 170, 3, 1)),
    ("win_top_left", (120, 160), (48, 64), (0, 0, 40, 30), None),
    ("win_bottom_right", (120, 160), (48, 64), (119, 89, 41, 31), None),
    ("win_left_edge", (121, 161), (40, 40), (0, 33, 20, 50), None),
    ("win_right_edge", (121, 161), (40, 40), (140, 33, 21, 50), None),
    ("win_top_edge", (121, 161), (40, 40), (31, 0, 47, 19), None),
    ("win_bottom_edge", (121, 161), (40, 40), (31, 102, 47, 19), None),
    ("win_1px_corner", (120, 160), (3, 3), (0, 0, 1, 1), None),
    ("win_1px_far_corner", (120, 160), (3, 3), (159, 119, 1, 1), None),
    ("win_1px_inside", (120, 160), (2, 5), (77, 51, 1, 1), None),
    ("win_odd_offset", (120, 160), (96, 96), (37, 21, 55, 43), None),
    ("win_row", (120, 160), (8, 96), (13, 57, 101, 1), None),
    ("win_col", (120, 160), (96, 8), (91, 3, 1, 99), None),
    ("win_small_frame", (3, 7), (6, 6), (1, 1, 5, 2), None),
]


def _cases():
    cases = []
    for name, hw, HW, window, form in _SHAPES:
        for layout in LAYOUTS:
            cases.append(("%s_%s" % (layout, name), layout, 700 + len(cases), hw, HW, window, form))
    return cases


CASES = _cases()


def raw_frame(seed, fh, fw):
    """Noise for even seeds, a noisy diagonal gradient (edges in both directions for the edge-aware choice) for odd ones."""
    rs = np.random.RandomState(seed)
    if seed % 2 == 0:
        return rs.randint(0, 256, (fh, fw)).astype(np.uint8)
    r, c = np.meshgrid(np.arange(fh), np.arange(fw), indexing="ij")
    g = (3 * r + 5 * c + ((r // 7 + c // 11) % 2) * 90) % 256
    return np.clip(g + rs.randint(-12, 13, (fh, fw)), 0, 255).astype(np.uint8)


def case_input(case):
    """The case's raw frame as the library takes it: a contiguous numpy array, or a view into a larger surface."""
    _, _, seed, (fh, fw), _, _, form = case
    raw = raw_frame(seed, fh, fw)
    if form is None:
        return raw
    _, SH, SW, y0, x0 = form
    surface = np.random.RandomState(seed + 1).randint(0, 256, (SH, SW)).astype(np.uint8)
    surface[y0:y0 + fh, x0:x0 + fw] = raw
    return surface[y0:y0 + fh, x0:x0 + fw]


def window_of(case):
    """(x0, y0, w, h) of the converted frame the case resizes."""
    _, _, _, (fh, fw), _, window, _ = case
    return window if window is not None else (0, 0, fw, fh)


def encode_cases():
    cases = []
    shapes = [  # name, (fh, fw), window, region, quality, sampling
        ("whole", (480, 640), None, None, 95, "420"),
        ("whole_odd", (241, 323), None, None, 75, "422"),
        ("whole_444", (97, 131), None, None, 90, "444"),
        ("tiny", (2, 5), None, None, 95, "420"),
        ("window", (240, 320), (37, 21, 155, 101), None, 95, "420"),
        ("window_region", (240, 320), (37, 21, 155, 101), (9, 3, 61, 47), 50, "444"),
        ("region_edge", (121, 161), None, (140, 100, 21, 21), 85, "422"),
        ("region_1px", (121, 161), None, (0, 120, 1, 1), 95, "420"),
        ("fullhd", (1080, 1920), None, None, 95, "420"),
    ]
    for k, (name, (fh, fw), window, region, q, s) in enumerate(shapes):
        for j, layout in enumerate(LAYOUTS if name != "fullhd" else ("bayer_rg", "bayer_gb_ea")):
            cases.append({"name": "%s_%s" % (layout, name), "layout": layout, "seed": 900 + 10 * k + j, "fh": fh, "fw": fw,
                          "window": window, "region": region, "quality": q, "sampling": s})
    return cases


ENCODE_CASES = encode_cases()


def encode_image(c, to_bgr):
    """The BGR image cv2.imencode encodes for case c, given a conversion to_bgr(raw, layout) (cv2's, or the oracle's)."""
    img = to_bgr(raw_frame(c["seed"], c["fh"], c["fw"]), c["layout"])
    for win in (c["window"], c["region"]):
        if win is not None:
            x0, y0, w, h = win
            img = img[y0:y0 + h, x0:x0 + w]
    return np.ascontiguousarray(img)

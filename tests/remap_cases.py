"""Seeded frames and remap maps for the goldens of tests/golden/make_golden_remap.py (cv2.cvtColor, cv2.remap INTER_LINEAR, crop,
cv2.resize INTER_LINEAR) and the tests.

A case is a dict: the inner frame (layout, seed, (fh, fw), `inner`: a window of it the maps address, or None), the maps (`map`:
(kind, mw, mh), `form`), the window of the remapped image (`view`, None for all of it) and the resize target (W, H).  The maps
are computed in numpy from seeds and fixed K, D values, with arithmetic only (no cv2 where the tests run):
  undistort  the pinhole model initUndistortRectifyMap states (k1, k2, p1, p2, k3), camera matrix from the sizes;
  fisheye    the equidistant model of cv2.fisheye (k1..k4), atan computed by halving and a series (basic operations only);
  random     coordinates inside and around the frame, with NaN, +-inf, +-1e9, 1e6 and half-way entries;
  grid64     every multiple of 1/64 as a fraction along both axes, so every code and every rounding tie appears;
  junk       fixed maps of random (x, y) around the frame and random 16-bit map2 (junk above the 10 code bits);
  cv2fixed   cv2.initUndistortRectifyMap(..., CV_16SC2)'s own fixed maps, stored in the golden file (fp64 rounding of its own).
form: "float2" (two float32 planes), "c2" (one float32 [h, w, 2]), "convert" (the fixed maps cv2.convertMaps makes of the float
maps) or "fixed" (junk, cv2fixed)."""
import numpy as np

import bayer_cases as bc
import layout_cases as lc

YUV420 = ("nv12", "nv21", "i420", "yv12")
LAYOUTS = ("bgr",) + YUV420 + ("rgb", "bgra", "rgba", "gray", "rgb_chw", "yuyv", "uyvy", "yvyu") + bc.LAYOUTS
CODES = {"nv12": "COLOR_YUV2BGR_NV12", "nv21": "COLOR_YUV2BGR_NV21", "i420": "COLOR_YUV2BGR_I420", "yv12": "COLOR_YUV2BGR_YV12",
         "rgb": "COLOR_RGB2BGR", "bgra": "COLOR_BGRA2BGR", "rgba": "COLOR_RGBA2BGR", "gray": "COLOR_GRAY2BGR",
         "rgb_chw": "COLOR_RGB2BGR", "yuyv": "COLOR_YUV2BGR_YUYV", "uyvy": "COLOR_YUV2BGR_UYVY", "yvyu": "COLOR_YUV2BGR_YVYU"}
CODES.update(bc.CODES)
D5 = (-0.28, 0.09, 0.001, -0.002, 0.0)           # k1, k2, p1, p2, k3
D4 = (0.1, -0.05, 0.01, -0.002)                  # fisheye k1..k4
FULL_BYTES = 4 * 1024                            # outputs up to this size are stored whole, larger ones as SHA-256
# convertMaps' edge values (x; y is 0): NaN, +-inf, +-1e9 -> (-32768, code 0); 1e6 -> 32767; 1048575.875 -> 32767, code 28;
# half-way fractions round to even
EDGE_VALUES = np.array([np.nan, np.inf, -np.inf, 1e9, -1e9, 1e6, -1e6, 1048575.875, 2.5 / 32, 3.5 / 32, -0.5 / 32, 1.5 / 32,
                        -1.5 / 32, 70000.0, -70000.0, 1023.984375, -1.0 / 64, 32767.0, -32768.0, 1e-30], np.float32)


def _case(name, layout, size, mp, form="float2", view=None, target=(64, 48), inner=None):
    return {"name": name, "layout": layout, "size": size, "map": mp, "form": form, "view": view, "target": target,
            "inner": inner}


def _cases():
    cases = []
    for layout in LAYOUTS:
        cases.append(_case(layout + "_undistort", layout, (76, 98), ("undistort", 98, 76)))
        cases.append(_case(layout + "_convert_window", layout, (76, 98), ("undistort", 98, 76), "convert", (5, 7, 80, 60),
                           (352, 352)))
    cases += [
        _case("bayer_gr_ea_inner_window", "bayer_gr_ea", (76, 98), ("fisheye", 90, 66), inner=(3, 5, 90, 66)),
        _case("bayer_bg_inner_window", "bayer_bg", (76, 98), ("undistort", 61, 41), "convert", inner=(37, 21, 55, 43)),
        _case("bgr_inner_crop", "bgr", (120, 160), ("undistort", 100, 70), inner=(31, 17, 100, 70)),
        _case("nv12_inner_crop", "nv12", (120, 160), ("undistort", 100, 70), "c2", inner=(30, 18, 100, 70)),
        _case("bgr_float2", "bgr", (120, 160), ("undistort", 160, 120), "float2", target=(128, 96)),
        _case("bgr_c2", "bgr", (120, 160), ("undistort", 160, 120), "c2", target=(128, 96)),
        _case("bgr_convert", "bgr", (120, 160), ("undistort", 160, 120), "convert", target=(128, 96)),
        _case("bgr_cv2fixed", "bgr", (120, 160), ("cv2fixed", 160, 120), "fixed", target=(128, 96)),
        _case("nv12_cv2fixed", "nv12", (120, 160), ("cv2fixed", 160, 120), "fixed", target=(96, 128)),
        _case("nv12_fisheye", "nv12", (120, 160), ("fisheye", 160, 120), "float2"),
        _case("bayer_rg_fisheye", "bayer_rg", (121, 161), ("fisheye", 161, 121), "c2"),
        _case("bgr_fisheye_convert", "bgr", (120, 160), ("fisheye", 160, 120), "convert", target=(352, 352)),
        _case("bgr_random", "bgr", (30, 40), ("random", 50, 40), "float2"),
        _case("gray_random", "gray", (31, 41), ("random", 45, 37), "c2"),
        _case("yuyv_random_convert", "yuyv", (30, 40), ("random", 50, 40), "convert"),
        _case("bayer_gb_random", "bayer_gb", (31, 41), ("random", 50, 40), "float2"),
        _case("bgr_grid64", "bgr", (40, 50), ("grid64", 128, 128), "float2", target=(128, 128)),
        _case("i420_grid64", "i420", (40, 50), ("grid64", 128, 128), "convert", target=(96, 80)),
        _case("bgr_junk", "bgr", (50, 60), ("junk", 40, 40), "fixed", target=(40, 40)),
        _case("rgba_junk", "rgba", (50, 60), ("junk", 40, 40), "fixed"),
        _case("bgr_map_smaller", "bgr", (120, 160), ("undistort", 30, 20), target=(352, 352)),
        _case("rgb_chw_map_larger", "rgb_chw", (30, 40), ("undistort", 300, 200), target=(160, 96)),
        _case("bgr_px1x1", "bgr", (1, 1), ("random", 5, 4), target=(4, 4)),
        _case("gray_px1x1", "gray", (1, 1), ("random", 3, 3)),
        _case("bayer_bg_px1x1", "bayer_bg", (1, 1), ("random", 3, 3)),
        _case("bgr_odd", "bgr", (23, 37), ("undistort", 37, 23), target=(29, 37)),
        _case("rgb_odd", "rgb", (177, 333), ("undistort", 333, 177), target=(352, 352)),
        _case("bgr_win_1px_corner", "bgr", (120, 160), ("undistort", 160, 120), view=(0, 0, 1, 1), target=(3, 3)),
        _case("bgr_win_far_corner", "bgr", (120, 160), ("undistort", 160, 120), view=(159, 119, 1, 1), target=(2, 5)),
        _case("bgr_win_edge", "bgr", (120, 160), ("undistort", 160, 120), view=(100, 80, 60, 40), target=(96, 64)),
        _case("nv21_win_odd", "nv21", (120, 160), ("undistort", 160, 120), view=(37, 21, 55, 43), target=(96, 96)),
        _case("bgr_upscale", "bgr", (120, 160), ("undistort", 20, 15), target=(128, 96)),
        _case("bgr_identity_target", "bgr", (120, 160), ("undistort", 160, 120), view=(11, 13, 101, 77), target=(101, 77)),
        _case("bgr_fullhd", "bgr", (1080, 1920), ("undistort", 1920, 1080), target=(352, 352)),
        _case("nv12_fullhd", "nv12", (1080, 1920), ("undistort", 1920, 1080), "convert", target=(352, 352)),
        _case("bayer_bg_fullhd", "bayer_bg", (1080, 1920), ("fisheye", 1920, 1080), target=(352, 352)),
    ]
    for k, c in enumerate(cases):
        c["seed"] = 1200 + k
    return cases


CASES = _cases()


def frame(layout, seed, fh, fw):
    """A seeded frame of `layout` in the form resize_frames takes: BGR [h, w, 3], cv2's single 4:2:0 buffer, the strided and
    4:2:2 layouts' arrays, a raw Bayer frame."""
    if layout in bc.LAYOUTS:
        return bc.raw_frame(seed, fh, fw)
    rs = np.random.RandomState(seed)
    shape = ((fh, fw, 3) if layout == "bgr" else (fh * 3 // 2, fw) if layout in YUV420 else lc.frame_shape(layout, fh, fw))
    return rs.randint(0, 256, shape).astype(np.uint8)


def case_frame(c):
    return frame(c["layout"], c["seed"], *c["size"])


def inner_size(c):
    """(w, h) of the image the maps address: the inner window, else the frame."""
    fh, fw = c["size"]
    return (c["inner"][2], c["inner"][3]) if c["inner"] else (fw, fh)


def _atan(r):
    """atan(r) for r >= 0 with basic operations only (bit-stable across numpy builds): two halvings, then the series."""
    t = r / (1.0 + np.sqrt(1.0 + r * r))
    t = t / (1.0 + np.sqrt(1.0 + t * t))
    t2, s, term = t * t, np.zeros_like(t), t.copy()
    for n in range(40):
        s = s + term / (2 * n + 1)
        term = -term * t2
    return 4.0 * s


def float_maps(kind, mw, mh, w, h, seed):
    """(mx, my) float32 [mh, mw] of a map kind over a w x h image."""
    v, u = np.meshgrid(np.arange(mh, dtype=np.float64), np.arange(mw, dtype=np.float64), indexing="ij")
    if kind in ("undistort", "fisheye"):
        x, y = (u - 0.5 * (mw - 1)) / (0.6 * mw), (v - 0.5 * (mh - 1)) / (0.6 * mw)
        r2 = x * x + y * y
        if kind == "undistort":
            k1, k2, p1, p2, k3 = D5
            rad = 1.0 + k1 * r2 + k2 * r2 * r2 + k3 * r2 * r2 * r2
            xd, yd = x * rad + 2 * p1 * x * y + p2 * (r2 + 2 * x * x), y * rad + p1 * (r2 + 2 * y * y) + 2 * p2 * x * y
        else:
            r = np.sqrt(r2)
            th = _atan(r)
            t2 = th * th
            thd = th * (1.0 + D4[0] * t2 + D4[1] * t2 * t2 + D4[2] * t2 * t2 * t2 + D4[3] * t2 * t2 * t2 * t2)
            s = np.where(r > 0, thd / np.where(r > 0, r, 1.0), 1.0)
            xd, yd = x * s, y * s
        return ((0.6 * w * xd + 0.5 * (w - 1)).astype(np.float32), (0.6 * w * yd + 0.5 * (h - 1)).astype(np.float32))
    rs = np.random.RandomState(seed)
    if kind == "random":
        mx = rs.uniform(-3, w + 2, (mh, mw)).astype(np.float32)
        my = rs.uniform(-3, h + 2, (mh, mw)).astype(np.float32)
        special = np.array([np.nan, np.inf, -np.inf, 1e9, -1e9, 1e6, -1e6, 2.5 / 32, -0.5 / 32, -1.0, float(w), w - 0.5],
                           np.float32)
        for m in (mx, my):
            pick = rs.randint(0, mh * mw, mh * mw // 6)
            m.reshape(-1)[pick] = special[rs.randint(0, len(special), len(pick))]
        return mx, my
    if kind == "grid64":
        fx, fy = (u % 64) / 64.0, (v % 64) / 64.0
        bx, by = rs.randint(-2, w + 2, (mh // 64 + 1, mw // 64 + 1)), rs.randint(-2, h + 2, (mh // 64 + 1, mw // 64 + 1))
        ix, iy = bx[(v // 64).astype(int), (u // 64).astype(int)], by[(v // 64).astype(int), (u // 64).astype(int)]
        return (ix + fx).astype(np.float32), (iy + fy).astype(np.float32)
    raise ValueError(kind)


def junk_maps(mw, mh, w, h, seed):
    rs = np.random.RandomState(seed)
    xy = np.stack([rs.randint(-5, w + 5, (mh, mw)), rs.randint(-5, h + 5, (mh, mw))], -1).astype(np.int16)
    return xy, rs.randint(0, 65536, (mh, mw)).astype(np.uint16)


def case_maps(c, golden=None):
    """The case's maps in its form, as cv2.remap takes them: (map1, map2); map2 None for "c2".  "convert" uses the oracle's
    convertMaps (pinned to cv2's by the golden file); "cv2fixed" reads cv2's maps from the golden file."""
    import remap_oracle as ro
    kind, mw, mh = c["map"]
    w, h = inner_size(c)
    if kind == "junk":
        return junk_maps(mw, mh, w, h, c["seed"])
    if kind == "cv2fixed":
        return golden[c["name"] + "_map1"], golden[c["name"] + "_map2"]
    mx, my = float_maps(kind, mw, mh, w, h, c["seed"])
    if c["form"] == "float2":
        return mx, my
    if c["form"] == "c2":
        return np.stack([mx, my], -1), None
    return ro.convert_maps(mx, my)


def fixed_maps(c, golden=None):
    """The case's maps in cv2's fixed form (what the remap reads)."""
    import remap_oracle as ro
    m1, m2 = case_maps(c, golden)
    if m1.dtype == np.int16:
        return m1, m2
    return ro.convert_maps(m1[..., 0], m1[..., 1]) if m2 is None else ro.convert_maps(m1, m2)


def view_window(c):
    """(x0, y0, w, h) of the remapped image the case resizes."""
    return c["view"] or (0, 0, c["map"][1], c["map"][2])


# encode cases: (case name, quality, sampling, region of the view's window or None): cv2.imencode of cv2's remapped window
ENCODE_CASES = [("bgr_undistort", 95, "420", None), ("nv12_fisheye", 90, "444", None), ("bayer_rg_fisheye", 75, "422", (10, 7, 61, 47)),
                ("gray_random", 95, "420", None), ("bgr_win_edge", 85, "420", (3, 2, 40, 30)), ("yuyv_convert_window", 95, "420", None)]


def camera(w, h):
    """The camera matrix make_golden_remap.py gives cv2.initUndistortRectifyMap (with D5) for a cv2fixed case of a w x h image."""
    return np.array([[0.6 * w, 0, 0.5 * (w - 1)], [0, 0.6 * w, 0.5 * (h - 1)], [0, 0, 1]], np.float64)

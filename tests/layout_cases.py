"""Seeded source frames in the layouts yfv2_resize_strided_u8 and yfv2_resize_yuv422_u8 read, for the goldens of
tests/golden/make_golden_layouts.py (cv2.cvtColor(COLOR_*2BGR) + cv2.resize) and the tests.

Each case is (name, layout, seed, (h, w), (H, W), form): a frame of noise drawn from numpy's legacy RandomState (bit-stable across
numpy versions) in `layout`'s array form, resized to H x W.  form None: a contiguous frame.  ("crop", SH, SW, y0, x0): the h x w
window at (y0, x0) of a larger SH x SW frame of the same layout (x0 even, so 4:2:2 crops start on a macropixel), a view with the
surface's row (and, for rgb_chw, channel) stride.  ("chw4",): channels 1..3 of a [4, h, w] array.  ("chw_every_other",):
channels 0, 2, 4 of a [6, h, w] array, whose channel stride is 2*h*w.  Plus the bundled images converted by cv2 in the golden
file."""
import numpy as np

from layout_oracle import MACROPIXEL

LAYOUTS = ("rgb", "bgra", "rgba", "gray", "rgb_chw", "yuyv", "uyvy", "yvyu")
YUV422 = ("yuyv", "uyvy", "yvyu")
MODELZOO_FRAMES = ("000139", "000004")


def frame_shape(layout, h, w):
    """The array shape of an h x w frame in `layout`."""
    if layout == "gray":
        return (h, w)
    if layout == "rgb_chw":
        return (3, h, w)
    return (h, w, {"rgb": 3, "bgra": 4, "rgba": 4}.get(layout, 2))


def _cases():
    cases = []
    for k, layout in enumerate(LAYOUTS):
        even = layout in YUV422
        odd = (177, 334 if even else 333)
        shapes = [
            ("down", (1080, 1920) if k % 2 == 0 else (720, 1280), (352, 352), None),
            ("odd", odd, (352, 352), None),
            ("row_1xN", (1, 400), (352, 352), None),
            ("col_Nx1", (400, 2 if even else 1), (352, 352), None),
            ("identity", (352, 352), (352, 352), None),
            ("upscale", (12, 16), (960, 1280), None),
            ("t37x29", (480, 640), (29, 37), None),
            ("t96x160", odd, (96, 160), None),
            ("crop", (300, 400), (352, 352), ("crop", 480, 640, 37, 86)),
        ]
        if layout == "rgb_chw":
            shapes += [("chw4", (240, 320), (352, 352), ("chw4",)),
                       ("chw_every_other", (177, 333), (96, 160), ("chw_every_other",))]
        if even:
            shapes += [("identity_odd", odd, odd, None)]
        for name, hw, HW, form in shapes:
            cases.append(("%s_%s" % (layout, name), layout, 300 + len(cases), hw, HW, form))
    return cases


CASES = _cases()


def case_input(case):
    """The case's frame as the library takes it: a contiguous numpy array or a view into a larger one."""
    _, layout, seed, (h, w), _, form = case
    rs = np.random.RandomState(seed)

    def noise(shape):
        return rs.randint(0, 256, size=shape).astype(np.uint8)

    if form is None:
        return noise(frame_shape(layout, h, w))
    if form[0] == "crop":
        _, SH, SW, y0, x0 = form
        s = noise(frame_shape(layout, SH, SW))
        return s[:, y0:y0 + h, x0:x0 + w] if layout == "rgb_chw" else s[y0:y0 + h, x0:x0 + w]
    if form[0] == "chw4":
        return noise((4, h, w))[1:]
    return noise((6, h, w))[::2]


def from_bgr(bgr, layout):
    """A packed BGR frame in `layout` as cv2.cvtColor(COLOR_BGR2RGB / BGR2BGRA / BGR2RGBA / BGR2GRAY) gives it (alpha 255; grey
    with OpenCV's 14-bit fixed point (1868 B + 9617 G + 4899 R + 2^13) >> 14), and planar CHW RGB."""
    if layout == "gray":
        b, g, r = (bgr[..., k].astype(np.int64) for k in range(3))
        return ((1868 * b + 9617 * g + 4899 * r + (1 << 13)) >> 14).astype(np.uint8)
    if layout == "rgb":
        return np.ascontiguousarray(bgr[..., ::-1])
    if layout in ("bgra", "rgba"):
        c = bgr if layout == "bgra" else bgr[..., ::-1]
        return np.concatenate([c, np.full(bgr.shape[:2] + (1,), 255, np.uint8)], -1)
    if layout == "rgb_chw":
        return np.ascontiguousarray(bgr[..., ::-1].transpose(2, 0, 1))
    raise ValueError(layout)


def yuyv_from_planes(y, u, v):
    """The [h, w, 2] YUYV frame of a Y plane [h, w] and the U and V samples [h, w/2] of its macropixels."""
    h, w = y.shape
    mp = np.empty((h, w // 2, 4), np.uint8)
    mp[..., 0], mp[..., 1], mp[..., 2], mp[..., 3] = y[:, 0::2], u, y[:, 1::2], v
    return mp.reshape(h, w, 2)


def bundled(golden, frames, img, layout):
    """The bundled image `img` (BGR, tests/golden/frames_modelzoo.npz) in `layout` as cv2.cvtColor(COLOR_BGR2<LAYOUT>) gives it.
    4:2:2 comes from cv2's YUYV conversion stored as planes in the golden file (UYVY and YVYU hold the same samples); the rest is
    restated here.  The golden file pins each to cv2's bytes by `<img>_<layout>_in_sha256`."""
    if layout in YUV422:
        yuyv = yuyv_from_planes(golden[img + "_yuyv_y"], golden[img + "_yuyv_u"], golden[img + "_yuyv_v"])
        return repack_yuv422(yuyv, "yuyv", layout)
    return from_bgr(frames[img], layout)


def repack_yuv422(frame, src, dst):
    """A [h, w, 2] packed 4:2:2 frame in layout `src` with its bytes reordered into layout `dst` (same Y, U and V samples)."""
    h, w, _ = frame.shape
    mp = np.ascontiguousarray(frame).reshape(h, w // 2, 4)
    out = np.empty_like(mp)
    for a, b in zip(MACROPIXEL[src], MACROPIXEL[dst]):
        out[..., b] = mp[..., a]
    return out.reshape(h, w, 2)

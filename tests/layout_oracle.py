"""CPU restatement (test infrastructure) of cv2.cvtColor(frame, COLOR_<LAYOUT>2BGR) followed by the resize of oracle/resize.py,
for every layout resize_frames takes.  RGB, BGRA / RGBA, grey and planar RGB are channel moves.  Packed YUV 4:2:2 (YUYV, UYVY,
YVYU) is converted with the BT.601 fixed point of tests/yuv_oracle.py (cv2 uses the same one as for 4:2:0), the U and V of each
pixel being those of its two-pixel macropixel.  Pinned to outputs of the real cv2.cvtColor + cv2.resize in
tests/golden/layout_cases.npz (tests/golden/make_golden_layouts.py)."""
import numpy as np

import yuv_oracle as yo
from oracle import resize as ore

# where the first Y, the U, the second Y and the V of a macropixel sit in its 4 bytes
MACROPIXEL = {"yuyv": (0, 1, 2, 3), "uyvy": (1, 0, 3, 2), "yvyu": (0, 3, 2, 1)}


def yuv422_to_bgr(frame, layout):
    """[h, w, 2] packed 4:2:2 uint8 (w even) -> the [h, w, 3] BGR bytes cv2.cvtColor(COLOR_YUV2BGR_<LAYOUT>) returns."""
    frame = np.asarray(frame)
    h, w, _ = frame.shape
    mp = frame.reshape(h, w // 2, 4)
    oy0, ou, oy1, ov = MACROPIXEL[layout]
    y = np.stack([mp[..., oy0], mp[..., oy1]], -1).reshape(h, w)
    # yuv_oracle's 4:2:0 conversion shares chroma over 2x2 blocks: give it every row twice and keep one of each pair
    return yo.yuv420_to_bgr(y.repeat(2, 0), mp[..., ou], mp[..., ov])[::2]


def to_bgr(frame, layout):
    """Any layout of resize_frames -> the packed [h, w, 3] BGR frame cv2.cvtColor makes of it (4:2:0 as a single buffer or
    planes, as tests/yuv_oracle.py takes them)."""
    if layout in yo.LAYOUTS:
        return yo.yuv420_to_bgr(*yo.split(frame, layout))
    if layout in MACROPIXEL:
        return yuv422_to_bgr(frame, layout)
    frame = np.asarray(frame)
    if layout == "bgr":
        return frame
    if layout == "rgb":
        return frame[..., ::-1]
    if layout == "bgra":
        return frame[..., :3]
    if layout == "rgba":
        return frame[..., 2::-1]
    if layout == "gray":
        return np.repeat(frame[..., None], 3, -1)
    if layout == "rgb_chw":
        return frame[::-1].transpose(1, 2, 0)
    raise ValueError(layout)


def resize_planar(frame, layout, W, H):
    """The [3, H, W] planar uint8 network input of cv2.resize(cv2.cvtColor(frame, COLOR_<LAYOUT>2BGR), (W, H), INTER_LINEAR)."""
    return ore.resize_bgr_planar(to_bgr(frame, layout), W, H)

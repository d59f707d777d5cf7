"""CPU restatement (test infrastructure) of cv2.convertMaps(mx, my, CV_16SC2) and cv2.remap(img, map1, map2, INTER_LINEAR) with the
default BORDER_CONSTANT 0 of OpenCV 4.13 (x86), composed with the layout, YUV and Bayer oracles (the cv2.cvtColor before it) and
oracle/resize.py (the cv2.resize after it).  Pinned to outputs of the real cv2 in tests/golden/remap_cases.npz
(tests/golden/make_golden_remap.py).

convertMaps, per coordinate v: X = rint_half_even(fl32(v * 32)) as int32, INT32_MIN for NaN, +-inf and |v * 32| >= 2^31;
x0 = saturate_int16(X >> 5), fraction X & 31; code = 32 * (y fraction) + (x fraction).
remap, per pixel with map1 = (x0, y0), code k (map2 & 1023), i = k >> 5, j = k & 31: the four taps (x0, y0), (x0 + 1, y0),
(x0, y0 + 1), (x0 + 1, y0 + 1) weighted by cv2's 2-D table entry k (weight_table), a tap outside the image contributing 0, and
sat_u8((sum + 16384) >> 15) per channel."""
import numpy as np

import bayer_oracle as bo
import layout_oracle as lo
from oracle import resize as ore


def convert_maps(mx, my):
    """cv2.convertMaps(mx, my, cv2.CV_16SC2) of float32 maps: (map1 int16 [h, w, 2], map2 uint16 [h, w])."""
    def fixed(v):
        v = np.asarray(v, np.float32) * np.float32(32)
        ok = np.isfinite(v) & (np.abs(v) < np.float32(2.0 ** 31))
        r = np.where(ok, np.rint(np.where(ok, v, 0)).astype(np.int64), -2 ** 31)
        return np.clip(r >> 5, -32768, 32767), r & 31
    with np.errstate(over="ignore", invalid="ignore"):
        x0, j = fixed(mx)
        y0, i = fixed(my)
    return np.stack([x0, y0], -1).astype(np.int16), (32 * i + j).astype(np.uint16)


def weight_table():
    """cv2's initInterTab2D for INTER_LINEAR with 8-bit images: int64 [1024, 4], entry 32 i + j.  The products
    fl32(fl32(1 - i/32) * fl32(1 - j/32)) and so on, each rint(p * 32768); a sum other than 32768 is corrected at the minimum or
    maximum entry (scanned from index 3, strict < first, else strict >)."""
    t = np.zeros((1024, 4), np.int64)
    for i in range(32):
        for j in range(32):
            ay, ax = np.float32(i / 32), np.float32(j / 32)
            cy, cx = (np.float32(1) - ay, ay), (np.float32(1) - ax, ax)
            v = [int(np.rint(np.float32(np.float32(cy[a] * cx[b]) * np.float32(32768)))) for a in range(2) for b in range(2)]
            diff = sum(v) - 32768
            if diff:
                mk = Mk = 3
                for k in range(4):
                    if v[k] < v[mk]:
                        mk = k
                    elif v[k] > v[Mk]:
                        Mk = k
                v[Mk if diff < 0 else mk] -= diff
            t[32 * i + j] = v
    return t


_TABLE = weight_table()


def remap(img, map1, map2):
    """cv2.remap(img, map1, map2, cv2.INTER_LINEAR) of a [h, w, 3] uint8 image through fixed maps: [mh, mw, 3] uint8."""
    img = np.asarray(img)
    h, w = img.shape[:2]
    x0, y0 = map1[..., 0].astype(np.int64), map1[..., 1].astype(np.int64)
    wt = _TABLE[np.asarray(map2).astype(np.int64) & 1023]
    acc = np.zeros(map1.shape[:2] + (3,), np.int64)
    for k, (dy, dx) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
        yy, xx = y0 + dy, x0 + dx
        inside = (yy >= 0) & (yy < h) & (xx >= 0) & (xx < w)
        px = img[np.clip(yy, 0, h - 1), np.clip(xx, 0, w - 1)].astype(np.int64)
        acc += np.where(inside[..., None], px, 0) * wt[..., k][..., None]
    return np.clip((acc + (1 << 14)) >> 15, 0, 255).astype(np.uint8)


def inner_bgr(frame, layout, window=None):
    """cv2.cvtColor(frame, COLOR_<LAYOUT>2BGR) of a frame of any layout; for Bayer the window (x0, y0, w, h) of the converted whole
    frame, for the others the crop of the converted frame."""
    if layout in bo.LAYOUTS:
        fh, fw = np.asarray(frame).shape
        return bo.window_bgr(frame, layout, *(window or (0, 0, fw, fh)))
    bgr = np.asarray(lo.to_bgr(frame, layout))
    if window is not None:
        x0, y0, w, h = window
        bgr = bgr[y0:y0 + h, x0:x0 + w]
    return np.ascontiguousarray(bgr)


def remap_window(img, map1, map2, window):
    """cv2.remap(img, map1, map2, INTER_LINEAR)[y0:y0 + h, x0:x0 + w]."""
    x0, y0, w, h = window
    return np.ascontiguousarray(remap(img, map1[y0:y0 + h, x0:x0 + w], map2[y0:y0 + h, x0:x0 + w]))


def resize_planar(img, map1, map2, window, W, H):
    """The [3, H, W] network input of cv2.resize(cv2.remap(img, map1, map2, INTER_LINEAR)[window], (W, H), INTER_LINEAR)."""
    return ore.resize_bgr_planar(remap_window(img, map1, map2, window), W, H)

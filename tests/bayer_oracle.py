"""CPU restatement (test infrastructure) of cv2.cvtColor(raw, COLOR_Bayer??2BGR) and its edge-aware variant (COLOR_Bayer??2BGR_EA)
of OpenCV 4.13, in integers on the raw bytes, followed by the resize of oracle/resize.py.  Pinned to outputs of the real cv2 in
tests/golden/bayer_cases.npz (tests/golden/make_golden_bayer.py).

For an interior pixel (1 <= r <= fh - 2, 1 <= c <= fw - 2), U, D, L, R its 4 neighbours and UL .. DR its diagonals:
  own colour                                    the raw byte;
  at a G site, the colour of L / R              (L + R + 1) >> 1, the colour of U / D: (U + D + 1) >> 1;
  at an R or B site, the other of R and B       (UL + UR + DL + DR + 2) >> 2;
  at an R or B site, G                          bilinear: (U + D + L + R + 2) >> 2;
                                                edge-aware: |L - R| <= |U - D| ? (L + R + 1) >> 1 : (U + D + 1) >> 1.
Pixel (r, c) of the border is the interior pixel at (clamp(r, 1, fh - 2), clamp(c, 1, fw - 2)); a frame with fw < 3 or fh < 3
converts to zeros."""
import numpy as np

from oracle import resize as ore

# layout -> (red_x, red_y): the column and row parity of the red sites; cv2's code is COLOR_Bayer<XY>2BGR (_EA)
RED = {"bg": (0, 0), "gb": (1, 0), "rg": (1, 1), "gr": (0, 1)}
LAYOUTS = tuple("bayer_" + k for k in RED) + tuple("bayer_%s_ea" % k for k in RED)


def pattern(layout):
    """(red_x, red_y, edge_aware) of a layout name."""
    red_x, red_y = RED[layout[6:8]]
    return red_x, red_y, layout.endswith("_ea")


def to_bgr(raw, layout):
    """[fh, fw] uint8 raw Bayer frame -> the [fh, fw, 3] BGR bytes cv2.cvtColor gives it for the layout's code."""
    raw = np.asarray(raw)
    fh, fw = raw.shape
    out = np.zeros((fh, fw, 3), np.uint8)
    if fw < 3 or fh < 3:
        return out
    red_x, red_y, ea = pattern(layout)
    p = raw.astype(np.int32)
    c = p[1:-1, 1:-1]
    up, dn, lf, rt = p[:-2, 1:-1], p[2:, 1:-1], p[1:-1, :-2], p[1:-1, 2:]
    hor, ver = (lf + rt + 1) >> 1, (up + dn + 1) >> 1
    diag = (p[:-2, :-2] + p[:-2, 2:] + p[2:, :-2] + p[2:, 2:] + 2) >> 2
    g_rb = np.where(np.abs(lf - rt) <= np.abs(up - dn), hor, ver) if ea else (up + dn + lf + rt + 2) >> 2
    r, cc = np.meshgrid(np.arange(1, fh - 1), np.arange(1, fw - 1), indexing="ij")
    red_row, red_col = (r & 1) == red_y, (cc & 1) == red_x
    red, blue = red_row & red_col, ~red_row & ~red_col
    green = ~(red | blue)
    B = np.where(blue, c, np.where(red, diag, np.where(red_row, ver, hor)))
    G = np.where(green, c, g_rb)
    R = np.where(red, c, np.where(blue, diag, np.where(red_row, hor, ver)))
    inner = np.stack([B, G, R], -1).astype(np.uint8)
    rows = np.clip(np.arange(fh), 1, fh - 2) - 1
    cols = np.clip(np.arange(fw), 1, fw - 2) - 1
    return inner[rows][:, cols]


def window_bgr(raw, layout, x0, y0, w, h):
    """cv2.cvtColor(raw)[y0:y0 + h, x0:x0 + w]: a window of the converted WHOLE frame (not the conversion of a cropped raw)."""
    return to_bgr(raw, layout)[y0:y0 + h, x0:x0 + w]


def resize_planar(raw, layout, W, H, window=None):
    """The [3, H, W] planar uint8 network input of cv2.resize(cv2.cvtColor(raw, code)[window], (W, H), INTER_LINEAR); window
    (x0, y0, w, h), None for the whole frame."""
    bgr = to_bgr(raw, layout) if window is None else window_bgr(raw, layout, *window)
    return ore.resize_bgr_planar(np.ascontiguousarray(bgr), W, H)


def mosaic(bgr, layout):
    """The raw Bayer frame a sensor of the layout's pattern records of a [h, w, 3] BGR image: each pixel keeps the channel of its
    site."""
    bgr = np.asarray(bgr)
    h, w, _ = bgr.shape
    red_x, red_y, _ = pattern(layout)
    r, c = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    red_row, red_col = (r & 1) == red_y, (c & 1) == red_x
    ch = np.where(red_row & red_col, 2, np.where(~red_row & ~red_col, 0, 1))
    return np.take_along_axis(bgr, ch[..., None], 2)[..., 0].copy()

"""CPU restatement (test infrastructure) of cv2.cvtColor(frame, cv2.COLOR_YUV2BGR_NV12 / _NV21 / _I420 / _YV12) followed by the
resize of oracle/resize.py, what a caller with decoded video frames runs before test.py:35-37.  OpenCV's x86 build converts YUV
4:2:0 with its ITUR_BT_601 fixed point (limited range, 20 fractional bits, chroma of each 2x2 block not interpolated):

  uu = U[r >> 1][c >> 1] - 128,  vv = V[r >> 1][c >> 1] - 128,  y = max(0, Y[r][c] - 16) * 1220542,  half = 1 << 19
  B = sat_u8((y + half + 2116026 * uu) >> 20)
  G = sat_u8((y + half - 852492 * vv - 409993 * uu) >> 20)
  R = sat_u8((y + half + 1673527 * vv) >> 20)

Pinned to outputs of the real cv2.cvtColor / cv2.cvtColorTwoPlane + cv2.resize in tests/golden/yuv_cases.npz
(tests/golden/make_golden_yuv.py), including all 2^24 (y, u, v) triples."""
import numpy as np

from oracle import resize as ore

LAYOUTS = ("nv12", "nv21", "i420", "yv12")


def yuv420_to_bgr(y, u, v):
    """Y [h, w], U and V [h/2, w/2] uint8 -> the [h, w, 3] BGR bytes cv2.cvtColor returns."""
    y, u, v = (np.asarray(p).astype(np.int64) for p in (y, u, v))
    uu = u.repeat(2, 0).repeat(2, 1) - 128
    vv = v.repeat(2, 0).repeat(2, 1) - 128
    yy = np.maximum(0, y - 16) * 1220542 + (1 << 19)
    bgr = np.stack([yy + 2116026 * uu, yy - 852492 * vv - 409993 * uu, yy + 1673527 * vv], -1) >> 20
    return np.clip(bgr, 0, 255).astype(np.uint8)


def resize_yuv420_planar(y, u, v, W, H):
    """The [3, H, W] planar uint8 network input of cv2.resize(cv2.cvtColor(frame), (W, H), INTER_LINEAR), from the three planes."""
    return ore.resize_bgr_planar(yuv420_to_bgr(y, u, v), W, H)


def split(frame, layout):
    """(Y, U, V) numpy planes of a frame given as cv2's single [h*3/2, w] buffer or as its tuple of planes ((y, uv) for NV12 /
    NV21, (y, u, v) for I420 / YV12)."""
    if isinstance(frame, (tuple, list)):
        if layout in ("nv12", "nv21"):
            y, uv = (np.asarray(p) for p in frame)
            a, b = uv[:, 0::2], uv[:, 1::2]
            return (y, a, b) if layout == "nv12" else (y, b, a)
        return tuple(np.asarray(p) for p in frame)
    frame = np.asarray(frame)
    h, w = frame.shape[0] // 3 * 2, frame.shape[1]
    if layout in ("nv12", "nv21"):
        return split((frame[:h], frame[h:]), layout)
    flat, q = np.ascontiguousarray(frame).reshape(-1), (h // 2) * (w // 2)
    first, second = flat[h * w:h * w + q].reshape(h // 2, w // 2), flat[h * w + q:h * w + 2 * q].reshape(h // 2, w // 2)
    return (frame[:h], first, second) if layout == "i420" else (frame[:h], second, first)


def resize_frame_planar(frame, layout, W, H):
    return resize_yuv420_planar(*split(frame, layout), W, H)

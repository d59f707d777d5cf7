"""CPU restatement (test infrastructure) of the resize every input of the reference goes through:

    cv2.resize(img, (cfg["width"], cfg["height"]), interpolation=cv2.INTER_LINEAR)     # test.py:35, utils/datasets.py:107

on packed HWC uint8 BGR images.  OpenCV is a third-party dependency of the reference; this restates the fixed-point arithmetic its
x86 build applies to 8-bit three-channel images (pinned to outputs of the real cv2.resize in tests/golden/resize_cases.npz,
tests/golden/make_golden_resize.py):

  coefficients, per axis (source length n, target length m):  scale = n / m in double;  f = fl32((d + 0.5) * scale - 0.5) with the
    product and the difference rounded in double;  s = floor(f);  f = fl32(f - s);  weights c0 = rint(fl32(1 - f) * 2048),
    c1 = rint(f * 2048), round half to even.  Along x only: s < 0 gives (s, f) = (0, 0), then s >= n - 1 gives (n - 1, 0).
  horizontal pass, exact int:  S[x] = src[sx] * a0 + src[min(sx + 1, w - 1)] * a1 per channel.
  vertical pass:  rows r0 = clamp(sy, 0, h - 1), r1 = clamp(sy + 1, 0, h - 1) with the weights (b0, b1) of the unclamped sy;
    out = sat_u8((((S0 >> 4) * b0 >> 16) + ((S1 >> 4) * b1 >> 16) + 2) >> 2).
"""
import numpy as np


def coeffs(n, m, clamp_edges):
    """Source index and the two 11-bit weights of each of the m target positions along an axis of source length n."""
    d = np.arange(m, dtype=np.float64)
    f = ((d + 0.5) * (np.float64(n) / np.float64(m)) - 0.5).astype(np.float32)
    s = np.floor(f)
    f = (f - s).astype(np.float32)
    s = s.astype(np.int64)
    if clamp_edges:
        lo = s < 0
        f[lo], s[lo] = 0, 0
        hi = s >= n - 1
        f[hi], s[hi] = 0, n - 1
    c0 = np.rint((np.float32(1) - f) * np.float32(2048)).astype(np.int64)
    c1 = np.rint(f * np.float32(2048)).astype(np.int64)
    return s, c0, c1


def resize_bgr(img, W, H):
    """uint8 [h, w, 3] -> uint8 [H, W, 3], the bytes cv2.resize(img, (W, H), interpolation=cv2.INTER_LINEAR) returns."""
    img = np.asarray(img)
    assert img.dtype == np.uint8 and img.ndim == 3 and img.shape[2] == 3
    h, w, _ = img.shape
    sx, a0, a1 = coeffs(w, W, True)
    x1 = np.minimum(sx + 1, w - 1)
    sy, b0, b1 = coeffs(h, H, False)
    r0, r1 = np.clip(sy, 0, h - 1), np.clip(sy + 1, 0, h - 1)
    src = img.astype(np.int64)

    def horizontal(rows):
        return src[rows[:, None], sx[None, :]] * a0[None, :, None] + src[rows[:, None], x1[None, :]] * a1[None, :, None]

    v = (((horizontal(r0) >> 4) * b0[:, None, None]) >> 16) + (((horizontal(r1) >> 4) * b1[:, None, None]) >> 16)
    return np.clip((v + 2) >> 2, 0, 255).astype(np.uint8)


def resize_bgr_planar(img, W, H):
    """The [3, H, W] planar form the network consumes (test.py:36-37: res_img.transpose(2, 0, 1))."""
    return np.ascontiguousarray(resize_bgr(img, W, H).transpose(2, 0, 1))

"""CPU restatement (test infrastructure) of the two img_aug steps the device adds to contrast_and_brightness
(utils/datasets.py:39-61), on packed HWC uint8 BGR images:

  augment_hsv(img, r):  cv2.cvtColor(BGR2HSV) -> per-image LUTs on H, S, V (datasets.py:44-47) -> cv2.cvtColor(HSV2BGR)
    BGR2HSV, OpenCV's 8-bit integer path (hsv_shift 12): sdiv[i] = rint((255 << 12) / i), hdiv[i] = rint((180 << 12) / (6 i)),
      entry 0 = 0;  v = max, diff = v - min, s = (diff * sdiv[v] + 2048) >> 12;  h = g - b if v == r, b - r + 2 diff if v == g,
      else r - g + 4 diff;  h = (h * hdiv[diff] + 2048) >> 12, + 180 if negative.
    HSV2BGR, OpenCV 4.13's 8-bit path (x86): in fp32, h *= fl(6/180), s *= fl(1/255), v *= fl(1/255);  sector = floor(h) mod 6,
      f = h - floor(h);  tab = (v, v (1 - s), v fma(-s, f, 1), v fma(-s, 1 - f, 1));  sector table
      {{1,3,0},{1,0,2},{3,0,1},{0,2,1},{0,1,3},{2,1,0}} picks B, G, R;  out = fl(x * 255) truncated, except in the last
      (w mod 32) pixels of each row, which cv2 converts with scalar code that rounds half to even.  The fused 1 - s*f (one
      rounding) and the truncation are what make it exact: with separate roundings the vector path differs on 1,836 of the 2^24
      triples; with rounding everywhere on 12.4 M.
  random_resize(img, rw, rh):  cv2.resize(cv2.resize(img, (rw, rh)), (W, H)), both INTER_LINEAR (oracle/resize.py).

Pinned to cv2 4.13 by tests/golden/aug_hsv_cases.npz (tests/golden/make_golden_aug_hsv.py): digests over all 2^24 triples and the
reference's own functions on seeded images."""
import numpy as np

from oracle import aug as oaug
from oracle import resize as ores

HSV_GAINS = (0.0138, 0.678, 0.36)          # augment_hsv's defaults (datasets.py:39)
_F = np.float32
_SECTORS = np.array([[1, 3, 0], [1, 0, 2], [3, 0, 1], [0, 2, 1], [0, 1, 3], [2, 1, 0]])


def _tables():
    i = np.arange(256, dtype=np.float64)
    with np.errstate(divide="ignore"):
        sdiv = np.where(i > 0, np.rint((255 << 12) / i), 0).astype(np.int64)
        hdiv = np.where(i > 0, np.rint((180 << 12) / (6.0 * i)), 0).astype(np.int64)
    return sdiv, hdiv


SDIV, HDIV = _tables()


def bgr2hsv(img):
    """uint8 [..., 3] BGR -> uint8 [..., 3] HSV (H in 0..179): cv2.cvtColor(img, cv2.COLOR_BGR2HSV)."""
    x = np.asarray(img).astype(np.int64)
    b, g, r = x[..., 0], x[..., 1], x[..., 2]
    v = np.maximum(np.maximum(b, g), r)
    diff = v - np.minimum(np.minimum(b, g), r)
    s = (diff * SDIV[v] + 2048) >> 12
    h = np.where(v == r, g - b, np.where(v == g, b - r + 2 * diff, r - g + 4 * diff))
    h = (h * HDIV[diff] + 2048) >> 12
    h = np.where(h < 0, h + 180, h)
    return np.stack([h, s, v], -1).astype(np.uint8)


def _fnma(a, b, c):
    """fl32(c - a * b) with one rounding (fp64 holds the product of two fp32 values exactly)."""
    return (np.float64(c) - a.astype(np.float64) * b.astype(np.float64)).astype(_F)


def hsv2bgr(img):
    """uint8 [h, w, 3] HSV (any H byte) -> uint8 [h, w, 3] BGR: cv2.cvtColor(img, cv2.COLOR_HSV2BGR)."""
    x = np.asarray(img)
    w = x.shape[-2]
    tail = (np.arange(w) >= (w & ~31))[:, None]
    h = x[..., 0].astype(_F) * _F(6.0 / 180.0)
    s = x[..., 1].astype(_F) * _F(1.0 / 255.0)
    v = x[..., 2].astype(_F) * _F(1.0 / 255.0)
    fl = np.floor(h)
    f = h - fl
    sector = fl.astype(np.int64) % 6
    tab = np.stack([v, v * (_F(1) - s), v * _fnma(s, f, 1), v * _fnma(s, _F(1) - f, 1)], -1)
    out = np.take_along_axis(tab, _SECTORS[sector], -1) * _F(255)
    return np.clip(np.where(tail, np.rint(out), np.trunc(out)), 0, 255).astype(np.uint8)


def hsv_luts(r):
    """datasets.py:44-47 for gains r (hue, saturation, value): uint8 [3, 256]."""
    x = np.arange(0, 256, dtype=np.int16)
    return np.stack([((x * r[0]) % 180).astype(np.uint8), np.clip(x * r[1], 0, 255).astype(np.uint8),
                     np.clip(x * r[2], 0, 255).astype(np.uint8)])


def augment_hsv(img, r):
    """datasets.py:39-51 with the gains r = uniform(-1, 1, 3) * gains + 1 given: uint8 [h, w, 3] BGR."""
    lut = hsv_luts(r)
    hsv = bgr2hsv(img)
    return hsv2bgr(np.stack([lut[k][hsv[..., k]] for k in range(3)], -1))


def random_resize(img, rw, rh):
    """datasets.py:54-61 with the drawn size (rw, rh) given."""
    h, w, _ = np.asarray(img).shape
    return ores.resize_bgr(ores.resize_bgr(img, rw, rh), w, h)


def img_aug(img, alpha, beta, rw=None, rh=None, r=None):
    """img_aug (datasets.py:63-68) with random_resize (when rw is given) and augment_hsv (when r is given) enabled."""
    img = oaug.contrast_and_brightness(img, alpha, beta)
    if rw is not None:
        img = random_resize(img, rw, rh)
    if r is not None:
        img = augment_hsv(img, r)
    return img


def all_triples():
    """The 4096 x 4096 x 3 image whose pixels are the 2^24 byte triples (pixel k = (k >> 16, (k >> 8) & 255, k & 255))."""
    k = np.arange(1 << 24, dtype=np.uint32)
    return np.stack([k >> 16, (k >> 8) & 255, k & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)

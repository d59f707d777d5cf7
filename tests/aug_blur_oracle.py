"""CPU restatement (test infrastructure) of the reference's motion_blur (utils/datasets.py:18-37) with its draws given, on packed
HWC uint8 BGR images, in the arithmetic of cv2 4.13 (x86):

  taps(degree, angle):  cv2.warpAffine(np.diag(np.ones(degree)), cv2.getRotationMatrix2D((degree/2, degree/2), angle, 1),
    (degree, degree)) / degree, converted to fp32 as filter2D converts its kernel.
      M: cos / sin of angle * fl64(pi/180) with libm, fp64;  inverted as cv2.invertAffineTransform (D = 1 / (m00 m11 - m01 m10)).
      Destination pixel (x, y): X = (cvRound(iM01 y + iM02) * 1024) + 16 + cvRound(iM00 x * 1024)) >> 5, Y likewise (AB_BITS
      10, INTER_BITS 5); source pixel (X >> 5, Y >> 5), fractions (X & 31) / 32, (Y & 31) / 32.
      Bilinear weights in fp32, (1 - vy)(1 - vx), (1 - vy) vx, vy (1 - vx), vy vx; outside pixels are 0 (BORDER_CONSTANT);
      the value is the fp64 sum v00 w0 + v01 w1 + v10 w2 + v11 w3 in that order.
  filter2D(img, k):  anchor (k // 2, k // 2), BORDER_REFLECT_101 per channel; out = cvRound(chain) saturated, the chain being
    fp32 fused multiply-adds over the taps in row-major order, starting from 0 (zero taps change nothing).
  normalize(img):  cv2.normalize(img, img, 0, 255, NORM_MINMAX): smin / smax over all bytes of the image (every channel);
    scale = 255 * (1 / (smax - smin)) when smax - smin > DBL_EPSILON else 0, shift = 0 - smin * scale (fp64);
    out = cvRound(fmaf(x, fl32(scale), fl32(shift))) saturated.  A constant image becomes all zeros.

Fused fp32 operations are computed in fp64 and rounded once: with bytes and these taps (products of at most 32 significant bits,
partial sums under 2^9, no bit below 2^-36) the fp64 sum is exact.  Pinned to cv2 by tests/golden/aug_blur_cases.npz
(tests/golden/make_golden_aug_blur.py)."""
import math

import numpy as np

_F = np.float32
_PI = 3.1415926535897932384626433832795            # CV_PI
_DBL_EPSILON = np.finfo(np.float64).eps


def rotation_matrix(degree, angle):
    """cv2.getRotationMatrix2D((degree / 2, degree / 2), angle, 1) as six Python floats (libm cos / sin)."""
    c = degree / 2
    a = angle * (_PI / 180)
    al, be = math.cos(a), math.sin(a)
    return [al, be, (1 - al) * c - be * c, -be, al, be * c + (1 - al) * c]


def invert_affine(m):
    """cv2.invertAffineTransform of a 2 x 3 matrix (six floats)."""
    d = m[0] * m[4] - m[1] * m[3]
    d = 1.0 / d if d != 0 else 0.0
    a11, a22, a12, a21 = m[4] * d, m[0] * d, -m[1] * d, -m[3] * d
    return [a11, a12, -a11 * m[2] - a12 * m[5], a21, a22, -a21 * m[2] - a22 * m[5]]


def warp_coords(degree, angle):
    """The fixed-point source coordinates cv2.warpAffine computes for each destination pixel: int [degree, degree] X and Y in
    1/32 pixel (X >> 5 is the column, X & 31 the fraction)."""
    im = invert_affine(rotation_matrix(degree, angle))
    X = np.empty((degree, degree), np.int64)
    Y = np.empty((degree, degree), np.int64)
    for y in range(degree):
        x0 = round(float(im[1] * y + im[2]) * 1024) + 16            # Python's round() is half to even, as cvRound
        y0 = round(float(im[4] * y + im[5]) * 1024) + 16
        for x in range(degree):
            X[y, x] = (x0 + round(im[0] * x * 1024)) >> 5
            Y[y, x] = (y0 + round(im[3] * x * 1024)) >> 5
    return X, Y


def warped_kernel(degree, angle):
    """cv2.warpAffine(np.diag(np.ones(degree)), M, (degree, degree)): float64 [degree, degree]."""
    src = np.eye(degree)
    X, Y = warp_coords(degree, angle)
    out = np.zeros((degree, degree))
    for y in range(degree):
        for x in range(degree):
            sx, sy = int(X[y, x] >> 5), int(Y[y, x] >> 5)
            vx, vy = _F((X[y, x] & 31) / 32), _F((Y[y, x] & 31) / 32)
            w = [(_F(1) - vy) * (_F(1) - vx), (_F(1) - vy) * vx, vy * (_F(1) - vx), vy * vx]
            v = [src[r, c] if 0 <= r < degree and 0 <= c < degree else 0.0
                 for r, c in ((sy, sx), (sy, sx + 1), (sy + 1, sx), (sy + 1, sx + 1))]
            s = 0.0
            for k in range(4):
                s = s + v[k] * float(w[k])
            out[y, x] = s
    return out


def taps(degree, angle):
    """The fp32 [degree, degree] kernel filter2D applies: warped_kernel / degree in fp64, then rounded to fp32."""
    return (warped_kernel(degree, angle) / degree).astype(_F)


def _reflect101(i, n):
    if n == 1:
        return np.zeros_like(i)
    i = np.abs(i)
    return np.where(i >= n, 2 * n - 2 - i, i)


def filter2d(img, k):
    """cv2.filter2D(img, -1, k) on uint8 [h, w, c] with the fp32 [ks, ks] kernel k (ks 2 or 3)."""
    img = np.asarray(img)
    h, w = img.shape[:2]
    ks = k.shape[0]
    a = ks // 2
    acc = np.zeros(img.shape, np.float64)
    for i in range(ks):
        rows = _reflect101(np.arange(h) + i - a, h)
        for j in range(ks):
            t = float(k[i, j])
            if t == 0.0:
                continue
            cols = _reflect101(np.arange(w) + j - a, w)
            v = img[rows][:, cols].astype(np.float64)
            acc = (v * t + acc).astype(_F).astype(np.float64)            # one fused rounding per tap
    return np.clip(np.rint(acc), 0, 255).astype(np.uint8)


def normalize_map(smin, smax):
    """cv2.normalize(NORM_MINMAX, 0..255) of a uint8 image with min smin and max smax, as a 256-entry byte map."""
    d = float(smax) - float(smin)
    scale = 255.0 * (1.0 / d) if d > _DBL_EPSILON else 0.0
    shift = 0.0 - float(smin) * scale
    x = np.arange(256, dtype=np.float64)
    y = (x * float(_F(scale)) + float(_F(shift))).astype(_F)            # fmaf: exact in fp64, one rounding
    return np.clip(np.rint(y), 0, 255).astype(np.uint8)


def normalize(img):
    img = np.asarray(img)
    return normalize_map(int(img.min()), int(img.max()))[img]


def motion_blur(img, degree, angle):
    """datasets.py:18-37 for an image that drew the blur (randint(1, 2) == 1) with the given degree and angle."""
    return normalize(filter2d(img, taps(degree, angle)))

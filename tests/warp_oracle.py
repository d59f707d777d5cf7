"""CPU restatement (test infrastructure) of cv2.warpAffine and cv2.warpPerspective with INTER_LINEAR and the default
BORDER_CONSTANT 0 of OpenCV 4.13 (x86): the fixed-point coordinates each computes per output pixel, then the sampling of
tests/remap_oracle.py (cv2.remap through CV_16SC2 maps), composed with the layout, YUV and Bayer oracles before it and
oracle/resize.py after it.  Pinned to outputs of the real cv2 in tests/golden/warp_cases.npz (tests/golden/make_golden_warp.py).

M is the destination -> source matrix (after inversion), row-major; all arithmetic is float64 element by element, in the order
written (numpy does not contract a * b + c):
  warpAffine       adelta[x] = cvRound((M[0] * x) * 1024), bdelta[x] = cvRound((M[3] * x) * 1024);
                   X0 = cvRound((M[1] * y + M[2]) * 1024) + 16, Y0 = cvRound((M[4] * y + M[5]) * 1024) + 16;
                   X = (X0 + adelta[x]) >> 5, Y = (Y0 + bdelta[x]) >> 5
  warpPerspective  W = (M[7] * y + M[8]) + M[6] * x, W = 32 / W if W else 0;
                   X = cvRound(clamp(((M[1] * y + M[2]) + M[0] * x) * W, INT_MIN, INT_MAX)), Y likewise with M[3..5]
  both             map1 = (sat_short(X >> 5), sat_short(Y >> 5)), map2 = (Y & 31) * 32 + (X & 31)
cvRound rounds half to even.  Inversion (without WARP_INVERSE_MAP): warpAffine's closed form, and cv2.invert(M, DECOMP_LU)'s
3x3 cofactor formula for warpPerspective (invert_affine, invert_perspective)."""
import numpy as np

import remap_oracle as ro
from oracle import resize as ore

AFFINE_LIMIT = 2.0 ** 30        # |every scaled term| must stay below this, so that the int32 sums cannot overflow


def invert_affine(m):
    """warpAffine's inversion of a 2x3 matrix (6 float64 values, row-major); the determinant's reciprocal is 0 when it is 0."""
    m = [float(v) for v in np.asarray(m, np.float64).reshape(-1)[:6]]
    D = m[0] * m[4] - m[1] * m[3]
    D = 1.0 / D if D != 0 else 0.0
    A11, A22 = m[4] * D, m[0] * D
    m[0] = A11
    m[1] *= -D
    m[3] *= -D
    m[4] = A22
    b1 = -m[0] * m[2] - m[1] * m[5]
    b2 = -m[3] * m[2] - m[4] * m[5]
    m[2], m[5] = b1, b2
    return np.array(m, np.float64)


def det3(m):
    return (m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6]))


def invert_perspective(m):
    """cv2.invert(M, DECOMP_LU) of a 3x3 float64 matrix: (ok, 9 values), all zero when the determinant is 0."""
    m = [float(v) for v in np.asarray(m, np.float64).reshape(-1)]
    d = det3(m)
    if d == 0:
        return False, np.zeros(9, np.float64)
    d = 1.0 / d
    t = [(m[4] * m[8] - m[5] * m[7]) * d, (m[2] * m[7] - m[1] * m[8]) * d, (m[1] * m[5] - m[2] * m[4]) * d,
         (m[5] * m[6] - m[3] * m[8]) * d, (m[0] * m[8] - m[2] * m[6]) * d, (m[2] * m[3] - m[0] * m[5]) * d,
         (m[3] * m[7] - m[4] * m[6]) * d, (m[1] * m[6] - m[0] * m[7]) * d, (m[0] * m[4] - m[1] * m[3]) * d]
    return True, np.array(t, np.float64)


def dst_to_src(M, inverse):
    """(perspective, the destination -> source matrix as 9 float64 values) of a 2x3 or 3x3 matrix given as cv2 takes it."""
    M = np.asarray(M, np.float64)
    perspective = M.shape == (3, 3)
    if not inverse:
        M = invert_perspective(M)[1] if perspective else invert_affine(M)
    m = np.zeros(9, np.float64)
    m[:M.size] = M.reshape(-1)
    return perspective, m


def _round(v):
    return np.rint(v).astype(np.int64)


def fixed_coords(m, perspective, x0, y0, w, h):
    """(X, Y) int64 [h, w]: the fixed-point source coordinates (1/32 pixel) of output pixels [y0, y0 + h) x [x0, x0 + w)."""
    x = np.arange(x0, x0 + w, dtype=np.float64)[None, :]
    y = np.arange(y0, y0 + h, dtype=np.float64)[:, None]
    if not perspective:
        ad, bd = _round((m[0] * x) * 1024.0), _round((m[3] * x) * 1024.0)
        X0, Y0 = _round((m[1] * y + m[2]) * 1024.0) + 16, _round((m[4] * y + m[5]) * 1024.0) + 16
        return (X0 + ad) >> 5, (Y0 + bd) >> 5
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        W = (m[7] * y + m[8]) + m[6] * x
        W = np.where(W != 0, 32.0 / np.where(W != 0, W, 1.0), 0.0)

        def coord(a, b, c):
            v = ((a * y + b) + c * x) * W
            v = np.where(v < 2147483647.0, v, 2147483647.0)               # std::min(INT_MAX, v): NaN -> INT_MAX
            v = np.where(-2147483648.0 < v, v, -2147483648.0)              # std::max(INT_MIN, v)
            return _round(v)
        return coord(m[1], m[2], m[0]), coord(m[4], m[5], m[3])


def warp_maps(m, perspective, x0, y0, w, h):
    """cv2's CV_16SC2 map1 and map2 of the window (x0, y0, w, h) of the warped image: what the warp samples through."""
    X, Y = fixed_coords(m, perspective, x0, y0, w, h)
    xy = np.stack([np.clip(X >> 5, -32768, 32767), np.clip(Y >> 5, -32768, 32767)], -1).astype(np.int16)
    return xy, ((Y & 31) * 32 + (X & 31)).astype(np.uint16)


def affine_fits(m, dw, dh):
    """Whether every scaled term of warpAffine stays below 2^30 in magnitude over a dw x dh output (the terms are linear in x
    and y, so the end points bound them)."""
    for x in (0.0, float(dw - 1)):
        if abs((m[0] * x) * 1024.0) >= AFFINE_LIMIT or abs((m[3] * x) * 1024.0) >= AFFINE_LIMIT:
            return False
    for y in (0.0, float(dh - 1)):
        if abs((m[1] * y + m[2]) * 1024.0) >= AFFINE_LIMIT or abs((m[4] * y + m[5]) * 1024.0) >= AFFINE_LIMIT:
            return False
    return True


def warp_window(img, M, dsize, window=None, inverse=False):
    """cv2.warpAffine / cv2.warpPerspective(img, M, dsize, INTER_LINEAR [| WARP_INVERSE_MAP])[y0:y0 + h, x0:x0 + w]."""
    perspective, m = dst_to_src(M, inverse)
    x0, y0, w, h = window or (0, 0) + tuple(dsize)
    return ro.remap(img, *warp_maps(m, perspective, x0, y0, w, h))


def resize_planar(img, M, dsize, window, W, H, inverse=False):
    """The [3, H, W] network input of cv2.resize(warp(img)[window], (W, H), INTER_LINEAR)."""
    return ore.resize_bgr_planar(warp_window(img, M, dsize, window, inverse), W, H)

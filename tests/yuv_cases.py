"""Seeded YUV 4:2:0 source frames for the goldens of tests/golden/make_golden_yuv.py (cv2.cvtColor + cv2.resize) and the tests.

Each case is (name, layout, seed, (h, w), (H, W), surface): a frame of noise drawn from numpy's legacy RandomState (bit-stable
across numpy versions), converted from `layout` and resized to H x W.  surface None: cv2's single [h*3/2, w] buffer.  Otherwise
surface = (SH, SW, y0, x0): the frame is the h x w window at the even offset (y0, x0) of a larger surface of SH luma rows SW bytes
apart, given as its planes; NV12 / NV21 keep one allocation with the UV rows after the SH luma rows (a decoder surface), I420 /
YV12 three separate planes.  Plus the colour cube (every (y, u, v) triple, cube_frame) and the bundled images, converted by
cv2.cvtColor(COLOR_BGR2YUV_I420) in the golden file."""
import numpy as np

CASES = [
    # each layout at least once
    ("nv12_fullhd", "nv12", 201, (1080, 1920), (352, 352), None),
    ("nv12_hd_640", "nv12", 202, (720, 1280), (640, 640), None),
    ("i420_vga", "i420", 203, (480, 640), (352, 352), None),
    ("nv21_500x376", "nv21", 204, (376, 500), (352, 352), None),
    ("yv12_518x334", "yv12", 205, (334, 518), (96, 160), None),
    # resize edge cases
    ("exact2x", "nv12", 206, (704, 704), (352, 352), None),
    ("identity", "i420", 207, (352, 352), (352, 352), None),
    ("upscale_big", "nv21", 208, (12, 16), (960, 1280), None),
    ("pixel_2x2", "yv12", 209, (2, 2), (5, 7), None),
    ("row_2xN", "yv12", 210, (2, 518), (352, 352), None),
    ("col_Nx2", "i420", 211, (334, 2), (352, 352), None),
    ("w37", "nv12", 212, (480, 640), (101, 37), None),
    ("w35", "nv21", 213, (200, 300), (33, 35), None),
    ("w11", "i420", 214, (76, 90), (13, 11), None),
    ("w97", "yv12", 215, (50, 70), (96, 97), None),
    # pitched and cropped sources
    ("nvdec_surface", "nv12", 216, (1080, 1920), (352, 352), (1088, 2048, 0, 0)),
    ("crop_two_plane", "nv21", 217, (400, 622), (352, 352), (720, 1280, 98, 214)),
    ("crop_three_plane", "i420", 218, (300, 400), (96, 160), (480, 640, 20, 34)),
    ("crop_three_plane_yv12", "yv12", 219, (226, 318), (352, 352), (334, 518, 106, 200)),
]

CUBE_FRAMES = 64          # NV12 512 x 512 frames, identity size, together every (y, u, v) in 0..255^3
MODELZOO_FRAMES = ("000139", "000004")


def cube_frame(k):
    """NV12 [768, 512] buffer k of the colour cube: chroma sample (i, j) is (u, v) = (i, j), and the four pixels of its 2x2 block
    carry y = 4k, 4k + 1 (top row), 4k + 2, 4k + 3 (bottom row)."""
    y = np.empty((512, 512), np.uint8)
    y[0::2, 0::2], y[0::2, 1::2], y[1::2, 0::2], y[1::2, 1::2] = 4 * k, 4 * k + 1, 4 * k + 2, 4 * k + 3
    i, j = np.meshgrid(np.arange(256, dtype=np.uint8), np.arange(256, dtype=np.uint8), indexing="ij")
    uv = np.stack([i, j], -1).reshape(256, 512)
    return np.concatenate([y, uv])


def case_input(case):
    """The case's frame as the library takes it: a single buffer, or a tuple of plane views into the case's surface."""
    _, layout, seed, (h, w), _, surface = case
    rs = np.random.RandomState(seed)
    if surface is None:
        return rs.randint(0, 256, size=(h * 3 // 2, w)).astype(np.uint8)
    SH, SW, y0, x0 = surface
    if layout in ("nv12", "nv21"):
        s = rs.randint(0, 256, size=(SH + SH // 2, SW)).astype(np.uint8)
        return s[y0:y0 + h, x0:x0 + w], s[SH + y0 // 2:SH + (y0 + h) // 2, x0:x0 + w]
    y = rs.randint(0, 256, size=(SH, SW)).astype(np.uint8)
    u = rs.randint(0, 256, size=(SH // 2, SW // 2)).astype(np.uint8)
    v = rs.randint(0, 256, size=(SH // 2, SW // 2)).astype(np.uint8)
    c = (slice(y0 // 2, (y0 + h) // 2), slice(x0 // 2, (x0 + w) // 2))
    return y[y0:y0 + h, x0:x0 + w], u[c], v[c]


def single_buffer(planes, layout):
    """cv2's single [h*3/2, w] buffer of a frame given as (y, uv) or (y, u, v) planes."""
    y = np.ascontiguousarray(planes[0])
    h, w = y.shape
    if layout in ("nv12", "nv21"):
        return np.concatenate([y, np.ascontiguousarray(planes[1])])
    u, v = planes[1], planes[2]
    first, second = (u, v) if layout == "i420" else (v, u)
    return np.concatenate([y.reshape(-1), np.ascontiguousarray(first).reshape(-1),
                           np.ascontiguousarray(second).reshape(-1)]).reshape(h * 3 // 2, w)


def i420_to_nv12(buf):
    """The NV12 buffer of an I420 buffer: the same luma, the U and V planes interleaved."""
    h, w = buf.shape[0] // 3 * 2, buf.shape[1]
    q = (h // 2) * (w // 2)
    flat = buf.reshape(-1)
    u, v = flat[h * w:h * w + q].reshape(h // 2, w // 2), flat[h * w + q:].reshape(h // 2, w // 2)
    return np.concatenate([buf[:h], np.stack([u, v], -1).reshape(h // 2, w)])

"""JPEG decode cases (tests/golden/make_golden_jpeg.py writes tests/golden/jpeg_cases.npz from them with cv2).

A supported case is (name, seed, (h, w), sampling, quality, optimize, restart, orientation, byte_order): a seeded image of that
size, cv2.imencode'd with IMWRITE_JPEG_QUALITY, _OPTIMIZE, _RST_INTERVAL and the sampling factor ("grey" encodes a one-channel
image), then, when orientation is not None, an EXIF APP1 carrying that orientation in the TIFF byte order "II" or "MM" inserted
after SOI.  The npz holds "jpg_<name>" (the file's bytes), and of cv2.imdecode(bytes, IMREAD_COLOR) its shape "shape_<name>", its
SHA-256 "sha_<name>" and, when it is at most FULL_BYTES, the frame itself "bgr_<name>" (so the goldens stay small; equals_golden
compares a decoded frame against whichever is there).

UNSUPPORTED lists the files the parser must refuse ("bad_<name>" in the npz): (name, parse code, a substring of the reason).
TRUNCATED_SCAN ("cut_<name>") is a file cut inside its entropy-coded data: the parser accepts it, the decode flags it."""
import hashlib

import numpy as np

FULL_BYTES = 1024

# name -> (luma h, luma v); chroma is 1x1
SAMPLINGS = {"444": (1, 1), "422": (2, 1), "420": (2, 2), "440": (1, 2), "411": (4, 1), "grey": (1, 1)}

CASES = []
_seed = 1000
for _s in SAMPLINGS:
    for _q in (1, 50, 75, 95, 100):
        for _opt in (0, 1):
            _seed += 1
            CASES.append(("q%d_%s_opt%d" % (_q, _s, _opt), _seed, (37, 53), _s, _q, _opt, 0, None, None))
for _s in SAMPLINGS:
    for (_h, _w) in ((1, 1), (1, 17), (17, 1), (8, 8), (15, 9), (16, 16), (31, 33), (37, 53), (333, 500)):
        _seed += 1
        CASES.append(("size%dx%d_%s" % (_h, _w, _s), _seed, (_h, _w), _s, 90, 0, 0, None, None))
for _s in SAMPLINGS:
    for _r in (0, 1, 7):
        _seed += 1
        CASES.append(("rst%d_%s" % (_r, _s), _seed, (45, 70), _s, 90, _r % 2, _r, None, None))
for _o in range(1, 9):
    for _order in ("II", "MM"):
        _seed += 1
        CASES.append(("exif%d_%s" % (_o, _order), _seed, (37, 53), "420" if _order == "II" else "422", 90, 0, 0, _o, _order))
CASES.append(("fullhd_420", 2001, (1080, 1920), "420", 90, 1, 0, None, None))

UNSUPPORTED = [
    ("progressive", -3, "progressive"),
    ("sof2", -3, "progressive"),
    ("sof3", -3, "lossless"),
    ("sof9", -3, "arithmetic"),
    ("bits12", -3, "12-bit"),
    ("comp4", -3, "4 components"),
    ("comp2", -3, "2 components"),
    ("two_scans", -3, "more than one scan"),
    ("adobe_rgb", -3, "RGB-coded"),
    ("sampling_22_21", -3, "sampling"),
    ("png", -3, "not a JPEG"),
    ("cut_header", -1, "truncated header"),
]

TRUNCATED_SCAN = "420_cut"


def mcus(case):
    """MCU count of a case's file."""
    _, _, (h, w), s, *_ = case
    hs, vs = SAMPLINGS[s] if s != "grey" else (1, 1)
    return -(-w // (8 * hs)) * -(-h // (8 * vs))


def segments(case):
    """Entropy-coded segments of a case's file: one per restart interval, one without."""
    r = case[6]
    return -(-mcus(case) // r) if r else 1


def digest(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def golden_shape(golden, name):
    return tuple(int(v) for v in golden["shape_" + name])


def equals_golden(golden, name, got):
    """True when the uint8 [h, w, 3] array `got` is cv2's frame of case `name`, byte for byte."""
    got = np.ascontiguousarray(got)
    if got.shape != golden_shape(golden, name):
        return False
    if "bgr_" + name in golden.files:
        return np.array_equal(got, golden["bgr_" + name])
    return np.array_equal(digest(got), golden["sha_" + name])


def image(seed, h, w, smooth=False):
    """Seeded BGR content: gradients, hard edges, noise and a saturated black / white checkerboard of 1-pixel cells (what drives
    the IDCT of a q100 file past 0..255); the noise only on images of at most 4096 pixels.  smooth: the gradients alone (the large
    frame).  Both keep the goldens small."""
    rs = np.random.RandomState(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.empty((h, w, 3), np.float64)
    for c in range(3):
        a, b, p = rs.uniform(-1, 1, 3)
        img[..., c] = 128 + 100 * np.sin(a * x / max(w, 1) * 6 + b * y / max(h, 1) * 6 + p * 3)
    if not smooth:
        img[:, w // 3:] += rs.randint(-40, 41, size=3)                                   # an edge
        img[h // 2:, :] = 255 - img[h // 2:, :]                                        # another
        noise = rs.randint(-24, 25, size=(h, w, 3))
        if h * w <= 4096:
            img += noise * (x[..., None] > w / 2)                                      # noise on the right half
        cb = (((y.astype(int) + x.astype(int)) & 1) * 255)[..., None]
        box = (y < h / 3) & (x < w / 3)
        img[box] = np.broadcast_to(cb, img.shape)[box]                                 # checkerboard in the top-left third
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)

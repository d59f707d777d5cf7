"""Cases of the JPEG encode goldens (tests/golden/make_golden_jpeg_encode.py): each output's frame is regenerated here from its
seed, so the golden stores only cv2's bytes (or, for the large outputs, their SHA-256 and length)."""
import numpy as np

SIZES = [(1, 1), (1, 2), (2, 1), (7, 9), (8, 8), (9, 8), (15, 17), (16, 16), (17, 16), (37, 53), (352, 352), (1920, 1080),
         (4097, 3)]                                   # (w, h): every w, h mod 8 and mod 16 class
QUALITIES = [1, 2, 10, 25, 49, 50, 51, 75, 90, 95, 99, 100, -5, 0, 101, 150]
SAMPLINGS = ["420", "422", "444"]
LARGE = 1 << 16                                       # outputs of more pixels are stored as SHA-256 + length
# cv2.cvtColor code of each layout ("gray": the 2-D frame itself, a one-component JPEG; "rgb_chw": transposed first)
CVT = {"bgr": None, "nv12": "COLOR_YUV2BGR_NV12", "nv21": "COLOR_YUV2BGR_NV21", "i420": "COLOR_YUV2BGR_I420",
       "yv12": "COLOR_YUV2BGR_YV12", "rgb": "COLOR_RGB2BGR", "bgra": "COLOR_BGRA2BGR", "rgba": "COLOR_RGBA2BGR", "gray": None,
       "rgb_chw": "COLOR_RGB2BGR", "yuyv": "COLOR_YUV2BGR_YUYV", "uyvy": "COLOR_YUV2BGR_UYVY", "yvyu": "COLOR_YUV2BGR_YVYU"}


def content(kind, w, h, seed, ch=3):
    """An h x w x ch uint8 image: seeded noise, flat 0 / 255, hard edges or a checkerboard"""
    rng = np.random.RandomState(seed)
    if kind == "noise":
        return rng.randint(0, 256, (h, w, ch), np.uint8)
    if kind in ("flat0", "flat255"):
        return np.full((h, w, ch), 0 if kind == "flat0" else 255, np.uint8)
    yy, xx = np.indices((h, w))
    if kind == "edges":
        m = ((xx * 3 + yy) // 11) % 2
    else:
        m = (xx // 3 + yy // 3) % 2
    lo, hi = rng.randint(0, 256, ch), rng.randint(0, 256, ch)
    return np.where(m[:, :, None] > 0, hi, lo).astype(np.uint8)


def frame(layout, w, h, kind, seed):
    """The raw frame of a case in `layout` (resize_frames' forms; 4:2:0 as cv2's [h*3/2, w] buffer)"""
    if layout in ("nv12", "nv21", "i420", "yv12"):
        return content(kind, w, h * 3 // 2, seed, 1)[:, :, 0].copy()
    if layout == "gray":
        return content(kind, w, h, seed, 1)[:, :, 0].copy()
    if layout in ("yuyv", "uyvy", "yvyu"):
        return content(kind, w, h, seed, 2)
    if layout in ("bgra", "rgba"):
        return content(kind, w, h, seed, 4)
    if layout == "rgb_chw":
        return np.ascontiguousarray(content(kind, w, h, seed).transpose(2, 0, 1))
    return content(kind, w, h, seed)


def cases():
    """(name, layout, content, w, h, seed, quality, sampling, restart, region (x0, y0, rw, rh) or None, photo or None)"""
    out = []

    def add(name, layout="bgr", kind="noise", w=37, h=53, seed=0, q=95, s="420", r=0, region=None, photo=None):
        out.append(dict(name=name, layout=layout, kind=kind, w=w, h=h, seed=seed, quality=q, sampling=s, restart=r, region=region,
                        photo=photo))

    for w, h in SIZES:
        add("size_%dx%d" % (w, h), w=w, h=h, seed=w * 7 + h)
        if w * h <= 352 * 352:
            for s in SAMPLINGS:
                add("size_%dx%d_%s_checker" % (w, h, s), kind="checker", w=w, h=h, s=s, q=75, seed=w + h)
                add("size_%dx%d_%s_grey" % (w, h, s), layout="gray", w=w, h=h, s=s, q=90, seed=w * h)
    for q in QUALITIES:
        for s in SAMPLINGS:
            add("quality_%d_%s" % (q, s), q=q, s=s, seed=q + 1000)
        add("quality_%d_grey" % q, layout="gray", w=17, h=16, q=q, seed=q + 2000)
    for kind in ("flat0", "flat255", "edges", "checker"):
        for s in SAMPLINGS:
            add("%s_%s" % (kind, s), kind=kind, w=40, h=33, s=s, q=100 if kind == "edges" else 95)
        add("%s_grey" % kind, layout="gray", kind=kind, w=41, h=30)
    for r in (1, 3, 1000):
        for s in SAMPLINGS:
            add("restart_%d_%s" % (r, s), w=37, h=53, s=s, r=r, seed=r)
            add("restart_%d_%s_352" % (r, s), w=352, h=352, s=s, r=r, seed=r + 1)
        add("restart_%d_grey" % r, layout="gray", w=37, h=53, r=r, seed=r + 2)
    for lay in CVT:
        add("layout_%s" % lay, layout=lay, w=36, h=52, seed=len(lay))
        add("layout_%s_q50_444" % lay, layout=lay, w=36, h=52, q=50, s="444", seed=len(lay) + 1)
    for lay in ("nv12", "i420", "yuyv", "uyvy"):
        for s in ("420", "422"):
            add("region_odd_%s_%s" % (lay, s), layout=lay, w=64, h=48, s=s, region=(3, 5, 29, 21))
            add("region_last_%s_%s" % (lay, s), layout=lay, w=64, h=48, s=s, region=(45, 37, 19, 11))
        add("region_1x1_%s" % lay, layout=lay, w=64, h=48, region=(63, 47, 1, 1))
    add("region_bgr_corner", w=50, h=40, region=(49, 0, 1, 40))
    for p in ("000004.jpg", "000139.jpg"):
        add("photo_%s" % p[:6], photo=p)
        add("photo_%s_q75_422_r5" % p[:6], photo=p, q=75, s="422", r=5)
        add("photo_%s_region" % p[:6], photo=p, q=90, region=(101, 33, 77, 151))
    return out


ROUNDTRIP = ["restart_3_420", "restart_1_422_352", "restart_1000_444", "restart_3_grey", "photo_000139_q75_422_r5",
             "size_37x53", "quality_100_420", "layout_nv12"]


def plan_error(kind, member, frames):
    """yfv2_jpeg_encode_plan of one whole-frame output per descriptor of `frames` (a ctypes array of the union member `member`),
    each wrapped as a yfv2_jpeg_enc_src of `kind`: (return code, yfv2_last_error()).  The plan reads no pixels."""
    import ctypes
    import yfv2_engine as eng
    srcs = (eng.JpegEncSrc * len(frames))()
    for s, f in zip(srcs, frames):
        s.kind = kind
        setattr(s.f, member, f)
        s.w, s.h = f.w, f.h
    L = eng.lib()
    mb, wb, ab = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_size_t()
    rc = L.yfv2_jpeg_encode_plan(srcs, len(frames), None, 0, ctypes.byref(mb), ctypes.byref(wb), None, ctypes.byref(ab))
    return rc, L.yfv2_last_error()

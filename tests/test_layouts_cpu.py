"""RGB, BGRA / RGBA, grey, planar RGB and packed YUV 4:2:2 frames, CPU side: the numpy restatement (tests/layout_oracle.py over
oracle/resize.py) against outputs of the real cv2.cvtColor + cv2.resize (tests/golden/layout_cases.npz), the descriptor checks
of yfv2_resize_strided_u8 and yfv2_resize_yuv422_u8 before any launch, and the refusals of resize_frames and detect_frames."""
import ctypes
import hashlib
import os

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import layout_cases as lc
import layout_oracle as lo


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "layout_cases.npz"))


@pytest.mark.parametrize("case", lc.CASES, ids=[c[0] for c in lc.CASES])
def test_oracle_matches_cv2(golden, case):
    name, layout, _, _, (H, W), _ = case
    frame = lc.case_input(case)
    assert np.array_equal(sha(frame), golden[name + "_in_sha256"]), "the seeded input generator changed"
    got = lo.resize_planar(frame, layout, W, H).transpose(1, 2, 0)
    if name + "_out" in golden:
        assert np.array_equal(got, golden[name + "_out"])
    assert np.array_equal(sha(got), golden[name + "_sha256"])


def test_cases_cover_every_layout_and_shape_class():
    for layout in lc.LAYOUTS:
        names = {c[0][len(layout) + 1:] for c in lc.CASES if c[1] == layout}
        assert {"down", "odd", "row_1xN", "col_Nx1", "identity", "upscale", "t37x29", "t96x160", "crop"} <= names, layout
    assert {c[0] for c in lc.CASES} >= {"rgb_chw_chw4", "rgb_chw_chw_every_other", "yuyv_identity_odd"}
    for case in lc.CASES:
        if case[1] in lc.YUV422:
            assert case[3][1] % 2 == 0 and (case[5] is None or case[5][4] % 2 == 0), case[0]


@pytest.mark.parametrize("layout", lc.LAYOUTS)
def test_oracle_gives_cv2s_result_on_the_bundled_images(golden, golden_dir, layout):
    """Every layout of the bundled images: the frame is cv2's conversion, and its 352 x 352 resize is cv2's; for the lossless
    layouts that is the stored network input of the BGR frame."""
    images = np.load(os.path.join(golden_dir, "images_modelzoo.npz"))
    frames = np.load(os.path.join(golden_dir, "frames_modelzoo.npz"))
    for img in lc.MODELZOO_FRAMES:
        frame = lc.bundled(golden, frames, img, layout)
        assert np.array_equal(sha(frame), golden["%s_%s_in_sha256" % (img, layout)]), (img, layout)
        got = lo.resize_planar(frame, layout, 352, 352)
        assert np.array_equal(sha(got.transpose(1, 2, 0)), golden["%s_%s_bgr352_sha256" % (img, layout)]), (img, layout)
        if layout not in lc.YUV422 + ("gray",):
            assert np.array_equal(got[None], images[img + "_u8"]), (img, layout)


def test_yuv422_oracle_pairs_each_pixel_with_its_macropixels_chroma():
    """A hand-made YUYV row: pixel 2j and 2j + 1 take U, V of macropixel j, never of a neighbour."""
    frame = np.array([[[100, 16], [100, 240], [100, 128], [100, 128]]], np.uint8)     # Y U Y V | Y U Y V
    bgr = lo.yuv422_to_bgr(frame, "yuyv")
    assert (bgr[0, 0] == bgr[0, 1]).all() and (bgr[0, 2] == bgr[0, 3]).all()
    assert bgr[0, 0, 0] < bgr[0, 2, 0] and bgr[0, 0, 2] > bgr[0, 2, 2]             # low U -> less blue; high V -> more red


def strided(*descs):
    import yfv2_engine as eng
    arr = (eng.StridedFrame * len(descs))()
    for a, (b, g, r, pitch, step, w, h) in zip(arr, descs):
        a.b, a.g, a.r, a.pitch, a.step, a.w, a.h = b, g, r, pitch, step, w, h
    return arr


def yuv422(*descs):
    import yfv2_engine as eng
    arr = (eng.Yuv422Frame * len(descs))()
    for a, (y, u, v, pitch, w, h) in zip(arr, descs):
        a.y, a.u, a.v, a.pitch, a.w, a.h = y, u, v, pitch, w, h
    return arr


def call_faults(make, good, fields, frame_faults):
    """Bad calls of one entry: the call-level faults, then each frame fault as the second frame of a two-frame batch, then one
    in the second launch's chunk."""
    fake = 0x1000
    dst = ctypes.c_void_p(fake)

    def bad(**kw):
        d = dict(zip(fields, good))
        d.update(kw)
        return tuple(d.values())

    calls = [(None, 1, 352, 352, dst), (make(good), 0, 352, 352, dst), (make(good), -1, 352, 352, dst),
             (make(good), 1, 352, 352, None), (make(good), 1, 0, 352, dst), (make(good), 1, 352, 0, dst),
             (make(good), 1, 352, 32769, dst), (make(good), 1, 32769, 352, dst)]
    calls += [(make(good, bad(**f)), 2, 352, 352, dst) for f in frame_faults]
    calls.append((make(*([good] * 130 + [bad(**frame_faults[0])])), 131, 352, 352, dst))
    return calls


def check_refusals(fn, name, calls):
    for i, args in enumerate(calls):
        assert fn(*args, None) == -1, i
        err = __import__("yfv2_engine").lib().yfv2_last_error()
        assert name in err, (i, err)
        if i >= 8:
            assert (b"frame 130" if i == len(calls) - 1 else b"frame 1") in err, (i, err)


def test_strided_abi_rejects_bad_descriptors_before_any_launch():
    import yfv2_engine as eng
    fake = 0x1000                                              # never dereferenced: every check runs on the host first
    good = (fake + 2, fake + 1, fake, 640 * 3, 3, 640, 480)
    faults = [dict(b=None), dict(g=None), dict(r=None), dict(w=0), dict(h=0), dict(w=-1), dict(h=-3),
              dict(step=0), dict(step=-3), dict(pitch=640 * 3 - 1), dict(step=4, pitch=640 * 4 - 1),
              dict(step=1 << 22, pitch=1 << 40)]                # step * w past 2^31
    check_refusals(eng.lib().yfv2_resize_strided_u8, b"resize_strided_u8",
                   call_faults(strided, good, ("b", "g", "r", "pitch", "step", "w", "h"), faults))


def test_yuv422_abi_rejects_bad_descriptors_before_any_launch():
    import yfv2_engine as eng
    fake = 0x1000
    good = (fake, fake + 1, fake + 3, 640 * 2, 640, 479)        # odd heights are allowed
    faults = [dict(y=None), dict(u=None), dict(v=None), dict(w=0), dict(h=0), dict(w=-2), dict(h=-1), dict(w=639),
              dict(pitch=640 * 2 - 1), dict(pitch=640)]
    check_refusals(eng.lib().yfv2_resize_yuv422_u8, b"resize_yuv422_u8",
                   call_faults(yuv422, good, ("y", "u", "v", "pitch", "w", "h"), faults))


def test_resize_frames_refuses_bad_frames_before_anything_runs():
    import yfv2_engine as eng
    rgb, chw, gray, yuyv = (np.zeros(s, np.uint8) for s in ((48, 64, 3), (3, 48, 64), (48, 64), (48, 64, 2)))
    cases = [
        ([rgb], "RGB", "layout"), ([rgb], "bgr24", "layout"), ([rgb], ["rgb", "yuv422"], "layout"), ([rgb], [None], "layout"),
        ([], "rgb", "no frames"), ([rgb, rgb], ["rgb"], "2 frames"),
        ([rgb.astype(np.float32)], "rgb", "uint8"),
        ([chw], "rgb", r"\[h, w, 3\]"), ([rgb], "bgra", r"\[h, w, 4\]"), ([np.zeros((48, 64, 4), np.uint8)], "rgb", r"\[h, w, 3\]"),
        ([rgb], "gray", r"\[h, w\]"), ([gray[None]], "gray", r"\[h, w\]"),
        ([rgb], "rgb_chw", r"\[3, h, w\]"), ([np.zeros((4, 48, 64), np.uint8)], "rgb_chw", r"\[3, h, w\]"),
        ([np.zeros((0, 64, 3), np.uint8)], "rgb", "h, w > 0"), ([np.zeros((3, 48, 0), np.uint8)], "rgb_chw", "h, w > 0"),
        ([rgb], "yuyv", r"\[h, w, 2\]"), ([yuyv[:, :63]], "uyvy", "even width"), ([np.zeros((5, 1, 2), np.uint8)], "yvyu", "even"),
        ([torch.zeros((48, 64, 2), dtype=torch.int16)], "yuyv", "uint8"),
        ([yuyv], "bgr", r"\[h, w, 3\]"), ([np.zeros((721, 640), np.uint8)], "nv12", r"\[h\*3/2, w\]"),
        # a bad frame after good ones of every kind: nothing is launched for the good ones either (no device is touched)
        ([rgb, np.zeros((72, 64), np.uint8), yuyv, rgb, chw, yuyv[:, :63]], ["bgr", "nv12", "yuyv", "rgb", "rgb_chw", "yuyv"],
         "frame 5"),
    ]
    for frames, layout, msg in cases:
        with pytest.raises(eng.Yfv2Error, match=msg):
            eng.resize_frames(frames, 352, 352, layout, device="cuda:0")
    with pytest.raises(eng.Yfv2Error, match="CUDA"):
        eng.resize_frames([rgb], 352, 352, "rgb", device="cpu")


def test_detect_frames_refuses_bad_layouts_and_shapes():
    import yfv2_engine as eng
    from utils import frames as uf
    model = torch.nn.Linear(1, 1)                              # never run: the frames are refused first
    cfg = {"width": 352, "height": 352}
    for frames, layout in [([np.zeros((48, 64, 3), np.uint8)], "hsv"), ([np.zeros((48, 63, 2), np.uint8)], "yuyv"),
                           ([np.zeros((48, 64), np.uint8)], ["gray", "gray"]), ([np.zeros((48, 64), np.uint8)], "rgb")]:
        with pytest.raises(eng.Yfv2Error):
            uf.detect_frames(model, frames, cfg, layout=layout)


def test_frame_size_of_every_layout():
    import yfv2_engine as eng
    assert len(eng.LAYOUTS) == 13 and set(lc.LAYOUTS) | {"bgr", "nv12", "nv21", "i420", "yv12"} == set(eng.LAYOUTS)
    for layout in eng.LAYOUTS:
        if layout in ("nv12", "nv21", "i420", "yv12"):
            frame = np.zeros((177 * 3 // 2 + 1, 334), np.uint8)[:-1]
            want = (176, 334)
        else:
            frame = np.zeros(lc.frame_shape(layout, 177, 334) if layout != "bgr" else (177, 334, 3), np.uint8)
            want = (177, 334)
        assert eng.frame_size(frame, layout) == want, layout

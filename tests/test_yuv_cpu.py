"""YUV 4:2:0 frames, CPU side: the numpy restatement (tests/yuv_oracle.py over oracle/resize.py) against outputs of the real
cv2.cvtColor + cv2.resize (tests/golden/yuv_cases.npz, including every (y, u, v) triple), the descriptor checks of
yfv2_resize_yuv420_u8 before any launch, and the refusals of the Python wrapper."""
import ctypes
import hashlib
import os

import numpy as np
import pytest

import yfv2  # noqa: F401
import yuv_cases as yc
import yuv_oracle as yo


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "yuv_cases.npz"))


@pytest.mark.parametrize("case", yc.CASES, ids=[c[0] for c in yc.CASES])
def test_oracle_matches_cv2(golden, case):
    name, layout, _, _, (H, W), _ = case
    y, u, v = yo.split(yc.case_input(case), layout)
    assert np.array_equal(sha(np.concatenate([np.ascontiguousarray(p).reshape(-1) for p in (y, u, v)])),
                          golden[name + "_in_sha256"]), "the seeded input generator changed"
    got = yo.resize_yuv420_planar(y, u, v, W, H).transpose(1, 2, 0)
    if name + "_out" in golden:
        assert np.array_equal(got, golden[name + "_out"])
    assert np.array_equal(sha(got), golden[name + "_sha256"])


def test_oracle_matches_cv2_on_the_whole_colour_cube(golden):
    """64 NV12 frames holding all 2^24 (y, u, v) triples, at identity size: the conversion alone, byte for byte."""
    seen = np.zeros(1 << 24, bool)
    for k in range(yc.CUBE_FRAMES):
        y, u, v = yo.split(yc.cube_frame(k), "nv12")
        got = yo.resize_yuv420_planar(y, u, v, 512, 512).transpose(1, 2, 0)
        assert np.array_equal(sha(got), golden["cube_%02d_sha256" % k]), k
        uu, vv = u.repeat(2, 0).repeat(2, 1), v.repeat(2, 0).repeat(2, 1)
        seen[(y.astype(np.int64) << 16) | (uu.astype(np.int64) << 8) | vv] = True
    assert seen.all()


def test_oracle_gives_cv2s_result_on_the_bundled_images(golden):
    """The bundled images as I420 (cv2.cvtColor(COLOR_BGR2YUV_I420)) and the NV12 derived from it give cv2's stored 352 x 352."""
    for name in yc.MODELZOO_FRAMES:
        i420 = golden[name + "_i420"]
        want = golden[name + "_bgr352"]
        assert np.array_equal(yo.resize_frame_planar(i420, "i420", 352, 352).transpose(1, 2, 0), want), name
        assert np.array_equal(yo.resize_frame_planar(yc.i420_to_nv12(i420), "nv12", 352, 352).transpose(1, 2, 0), want), name


def test_single_buffer_and_planes_split_alike():
    for case in yc.CASES:
        layout = case[1]
        frame = yc.case_input(case)
        planes = frame if isinstance(frame, tuple) else None
        buf = yc.single_buffer(planes, layout) if planes else frame
        for a, b in zip(yo.split(buf, layout), yo.split(frame, layout)):
            assert np.array_equal(a, b), case[0]


def yuv_descs(*descs):
    import yfv2_engine as eng
    arr = (eng.Yuv420Frame * len(descs))()
    for a, (yp, ypitch, up, vp, uvpitch, step, w, h) in zip(arr, descs):
        a.y, a.y_pitch, a.u, a.v, a.uv_pitch, a.uv_step, a.w, a.h = yp, ypitch, up, vp, uvpitch, step, w, h
    return arr


def test_abi_rejects_bad_descriptors_before_any_launch():
    import yfv2_engine as eng
    L = eng.lib()
    fake = 0x1000                                              # never dereferenced: every check runs on the host first
    dst = ctypes.c_void_p(fake)
    nv12 = (fake, 640, fake + 640 * 480, fake + 640 * 480 + 1, 640, 2, 640, 480)
    i420 = (fake, 640, fake + 4096, fake + 8192, 320, 1, 640, 480)

    def bad(**kw):
        d = dict(zip(("y", "y_pitch", "u", "v", "uv_pitch", "uv_step", "w", "h"), i420 if kw.pop("planar", False) else nv12))
        d.update(kw)
        return tuple(d.values())

    bad_calls = [
        (None, 1, 352, 352, dst),
        (yuv_descs(nv12), 0, 352, 352, dst),
        (yuv_descs(nv12), -1, 352, 352, dst),
        (yuv_descs(nv12), 1, 352, 352, None),
        (yuv_descs(nv12), 1, 0, 352, dst),
        (yuv_descs(nv12), 1, 352, 0, dst),
        (yuv_descs(nv12), 1, 352, 32769, dst),
        (yuv_descs(nv12), 1, 32769, 352, dst),
    ]
    frame_faults = [
        bad(y=None), bad(u=None), bad(v=None),
        bad(w=0), bad(h=0), bad(w=-2), bad(h=-2), bad(w=639), bad(h=479),
        bad(y_pitch=639),
        bad(uv_pitch=639),                                   # interleaved chroma needs w bytes per row
        bad(planar=True, uv_pitch=319),                      # planar chroma needs w / 2
        bad(uv_step=0), bad(uv_step=3), bad(planar=True, uv_step=-1),
    ]
    for f in frame_faults:
        bad_calls.append((yuv_descs(nv12, f), 2, 352, 352, dst))
    # a bad frame in the second launch's chunk (64 descriptors per launch)
    bad_calls.append((yuv_descs(*([nv12, i420] * 40 + [bad(h=7)])), 81, 352, 352, dst))
    for i, args in enumerate(bad_calls):
        assert L.yfv2_resize_yuv420_u8(*args, None) == -1, i
        assert b"resize_yuv420_u8" in L.yfv2_last_error(), (i, L.yfv2_last_error())
        if i >= 8:
            assert (b"frame 80" if i == len(bad_calls) - 1 else b"frame 1") in L.yfv2_last_error(), (i, L.yfv2_last_error())


def test_python_wrapper_refuses_bad_frames_before_copying():
    import yfv2_engine as eng
    nv12 = np.zeros((720, 640), np.uint8)
    cases = [
        ([nv12], "rgb", "layout"),
        ([nv12], "NV12", "layout"),
        ([], "nv12", "no frames"),
        ([nv12.astype(np.float32)], "nv12", "uint8"),
        ([np.zeros((720, 640, 1), np.uint8)], "nv12", "uint8"),
        ([np.zeros((721, 640), np.uint8)], "nv12", r"\[h\*3/2, w\]"),
        ([np.zeros((722, 640), np.uint8)], "i420", r"\[h\*3/2, w\]"),
        ([np.zeros((720, 641), np.uint8)], "nv21", r"\[h\*3/2, w\]"),
        ([np.zeros((0, 640), np.uint8)], "yv12", r"\[h\*3/2, w\]"),
        ([(np.zeros((480, 640), np.uint8),)], "nv12", "planes"),
        ([(np.zeros((480, 640), np.uint8),) * 3], "nv12", "planes"),
        ([(np.zeros((480, 640), np.uint8),) * 2], "i420", "planes"),
        ([(np.zeros((480, 640), np.uint8), np.zeros((240, 320), np.uint8))], "nv12", "chroma"),
        ([(np.zeros((479, 640), np.uint8), np.zeros((239, 640), np.uint8))], "nv12", "even"),
        ([(np.zeros((480, 640), np.uint8), np.zeros((240, 320), np.uint8), np.zeros((240, 321), np.uint8))], "i420", "chroma"),
        ([(np.zeros((480, 640), np.uint8), np.zeros((240, 640), np.int16))], "nv12", "uint8"),
    ]
    for frames, layout, msg in cases:
        with pytest.raises(eng.Yfv2Error, match=msg):
            eng.resize_yuv420(frames, 352, 352, layout, device="cuda:0")
    with pytest.raises(eng.Yfv2Error, match="CUDA"):
        eng.resize_yuv420([nv12], 352, 352, "nv12", device="cpu")


def test_detect_frames_sizes_yuv_frames_by_their_luma_plane():
    from utils import frames as uf
    assert uf._yuv420_size(np.zeros((1620, 1920), np.uint8)) == (1080, 1920)
    assert uf._yuv420_size((np.zeros((334, 500), np.uint8), np.zeros((167, 500), np.uint8))) == (334, 500)
    assert uf.resize_yuv420 is not None and uf.resize_bgr is not None

"""Raw-frame resize, CPU side: the numpy restatement (oracle/resize.py) against outputs of the real cv2.resize
(tests/golden/resize_cases.npz, frames_modelzoo.npz), argument checks of yfv2_resize_bgr_u8 (and of the JPEG encoder's plan on
the same frames) before any launch, and the host scale-back of detect_frames against test.py's own arithmetic."""
import ctypes
import hashlib
import os

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import jpeg_encode_cases as jc
import resize_cases as rc
from oracle import resize as ore


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


@pytest.mark.parametrize("case", rc.CASES, ids=[c[0] for c in rc.CASES])
def test_oracle_matches_cv2_resize(golden_dir, case):
    g = np.load(os.path.join(golden_dir, "resize_cases.npz"))
    name, _, _, _, (H, W) = case
    _, src = rc.case_input(case)
    assert np.array_equal(sha(src), g[name + "_in_sha256"]), "the seeded input generator changed"
    got = ore.resize_bgr(src, W, H)
    assert got.shape == (H, W, 3)
    if name + "_out" in g:
        assert np.array_equal(got, g[name + "_out"])
    assert np.array_equal(sha(got), g[name + "_sha256"])


def test_oracle_gives_the_stored_network_inputs_of_the_bundled_images(golden_dir):
    """cv2.imread + cv2.resize + transpose of img/000139.jpg and img/000004.jpg (test.py:34-37) are the *_u8 inputs every
    known-answer test uses."""
    frames = np.load(os.path.join(golden_dir, "frames_modelzoo.npz"))
    g = np.load(os.path.join(golden_dir, "images_modelzoo.npz"))
    for name in rc.MODELZOO_FRAMES:
        assert np.array_equal(ore.resize_bgr_planar(frames[name], 352, 352)[None], g[name + "_u8"]), name


def test_abi_rejects_bad_arguments_before_any_launch():
    import yfv2_engine as eng
    L = eng.lib()
    fake = 0x1000                                            # never dereferenced: every check runs on the host first
    dst = ctypes.c_void_p(fake)

    def frames(*descs):
        arr = (eng.Frame * len(descs))()
        for a, (data, w, h, pitch) in zip(arr, descs):
            a.data, a.w, a.h, a.pitch = data, w, h, pitch
        return arr

    ok = (fake, 640, 480, 1920)
    bad_calls = [
        (None, 1, 352, 352, dst),
        (frames(ok), 0, 352, 352, dst),
        (frames(ok), -1, 352, 352, dst),
        (frames(ok), 1, 352, 352, None),
        (frames(ok), 1, 0, 352, dst),
        (frames(ok), 1, 352, 0, dst),
        (frames(ok), 1, 32769, 352, dst),
        (frames(ok, (None, 640, 480, 1920)), 2, 352, 352, dst),
        (frames(ok, (fake, 0, 480, 1920)), 2, 352, 352, dst),
        (frames(ok, (fake, 640, 0, 1920)), 2, 352, 352, dst),
        (frames(ok, (fake, 640, 480, 1919)), 2, 352, 352, dst),          # pitch < 3 * w
        (frames(*([ok] * 200 + [(fake, 640, 480, -1)])), 201, 352, 352, dst),   # a bad frame in the second launch's chunk
    ]
    assert jc.plan_error(eng.JPEG_SRC_BGR, "bgr", frames(ok))[0] == 0
    for i, args in enumerate(bad_calls):
        assert L.yfv2_resize_bgr_u8(*args, None) == -1, i
        assert b"resize_bgr_u8" in L.yfv2_last_error(), (i, L.yfv2_last_error())
        if i >= 7:
            at = 200 if i == len(bad_calls) - 1 else 1
            assert b"frame %d" % at in L.yfv2_last_error(), (i, L.yfv2_last_error())
            code, err = jc.plan_error(eng.JPEG_SRC_BGR, "bgr", args[0])     # the JPEG encoder's plan refuses them too
            assert code == -1 and b"jpeg_encode_plan: output %d: frame" % at in err, (i, err)


def test_python_entry_points_refuse_bad_frames():
    import yfv2_engine as eng
    with pytest.raises(eng.Yfv2Error, match="uint8"):
        eng.resize_bgr([np.zeros((4, 4, 3), np.float32)], 32, 32, device="cuda:0")
    with pytest.raises(eng.Yfv2Error, match="uint8"):
        eng.resize_bgr([np.zeros((4, 4), np.uint8)], 32, 32, device="cuda:0")
    with pytest.raises(eng.Yfv2Error, match="CUDA"):
        eng.resize_bgr([np.zeros((4, 4, 3), np.uint8)], 32, 32, device="cpu")
    with pytest.raises(eng.Yfv2Error, match="no frames"):
        eng.resize_bgr([], 32, 32, device="cuda:0")


def test_scale_back_is_test_py_arithmetic():
    """test.py:57-68: scale_h, scale_w = h / cfg["height"], w / cfg["width"]; corners box[i] * scale in Python floats, drawn at
    int() of them."""
    from utils import frames as uf
    cfg = {"width": 352, "height": 352}
    rs = np.random.RandomState(3)
    rows = np.zeros((300, 6), np.float32)
    rows[:, :4] = rs.uniform(-20, 372, (300, 4))
    rows[:, 4] = rs.rand(300)
    rows[:, 5] = rs.randint(0, 80, 300)
    for h, w in ((1080, 1920), (334, 500), (480, 640), (17, 3)):
        got = uf.to_source_pixels(torch.from_numpy(rows), (h, w), cfg)
        corners = uf.int_corners(got)
        scale_h, scale_w = h / cfg["height"], w / cfg["width"]
        assert got.dtype == torch.float64
        for r, b, c in zip(got.tolist(), rows, corners.tolist()):
            box = torch.from_numpy(b).tolist()
            assert r == [box[0] * scale_w, box[1] * scale_h, box[2] * scale_w, box[3] * scale_h, box[4], box[5]]
            assert c == [int(box[0] * scale_w), int(box[1] * scale_h), int(box[2] * scale_w), int(box[3] * scale_h)]

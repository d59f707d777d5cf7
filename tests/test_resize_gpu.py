"""Raw-frame resize on the device (yfv2_resize_bgr_u8 through the C ABI) against the frozen cv2.resize outputs and the numpy
oracle, bit for bit; and detect_frames, raw frames to boxes in source pixels, against the test.py known answers."""
import hashlib
import os

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import resize_cases as rc
import synth
import yfv2_engine as eng
from oracle import resize as ore

pytestmark = pytest.mark.gpu


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def device_window(case):
    """The case's window as a CUDA view into its whole frame (a crop keeps the frame's row pitch)."""
    full, _ = rc.case_input(case)
    d = torch.from_numpy(full).cuda()
    win = case[3]
    if win is None:
        return d
    y0, x0, h, w = win
    return d[y0:y0 + h, x0:x0 + w]


def hwc(planar):
    return planar.permute(1, 2, 0).contiguous().cpu().numpy()


@pytest.mark.parametrize("case", rc.CASES, ids=[c[0] for c in rc.CASES])
def test_bit_exact_against_cv2_golden(golden_dir, case):
    g = np.load(os.path.join(golden_dir, "resize_cases.npz"))
    name, _, _, _, (H, W) = case
    out = eng.resize_bgr([device_window(case)], W, H)
    assert out.shape == (1, 3, H, W) and out.dtype == torch.uint8
    got = hwc(out[0])
    if name + "_out" in g:
        assert np.array_equal(got, g[name + "_out"])
    assert np.array_equal(sha(got), g[name + "_sha256"])


@pytest.mark.parametrize("H,W", [(352, 352), (96, 160)])
def test_mixed_size_batch_equals_per_frame_results(H, W):
    frames = [device_window(c) for c in rc.CASES]
    batch = eng.resize_bgr(frames, W, H)
    for i, f in enumerate(frames):
        assert torch.equal(batch[i], eng.resize_bgr([f], W, H)[0]), rc.CASES[i][0]
        assert np.array_equal(batch[i].cpu().numpy(), ore.resize_bgr_planar(f.cpu().numpy(), W, H)), rc.CASES[i][0]


def test_pitched_crop_equals_contiguous_copy():
    full = torch.from_numpy(rc.frame(7, (1080, 1920))).cuda()
    for (y0, x0, h, w) in [(0, 0, 1080, 1919), (131, 7, 517, 771), (1078, 1, 2, 1918), (3, 1917, 1077, 3)]:
        crop = full[y0:y0 + h, x0:x0 + w]
        assert crop.stride(0) == 1920 * 3 and not crop.is_contiguous()
        a = eng.resize_bgr([crop], 352, 352)
        b = eng.resize_bgr([crop.contiguous()], 352, 352)
        assert torch.equal(a, b), (y0, x0, h, w)
        # a host numpy crop (rows 5760 bytes apart) goes through the same path
        assert torch.equal(eng.resize_bgr([crop.cpu().numpy()], 352, 352), a)


def test_many_frames_span_several_launches():
    """More frames than one launch's descriptor chunk (128): every frame lands in its own slot."""
    rs = np.random.RandomState(9)
    frames = [rs.randint(0, 256, (rs.randint(1, 90), rs.randint(1, 90), 3)).astype(np.uint8) for _ in range(300)]
    out = eng.resize_bgr(frames, 37, 29).cpu().numpy()
    for i, f in enumerate(frames):
        assert np.array_equal(out[i], ore.resize_bgr_planar(f, 37, 29)), i


def test_bundled_frames_give_the_stored_network_inputs(golden_dir):
    frames = np.load(os.path.join(golden_dir, "frames_modelzoo.npz"))
    g = np.load(os.path.join(golden_dir, "images_modelzoo.npz"))
    out = eng.resize_bgr([frames[n] for n in rc.MODELZOO_FRAMES], 352, 352).cpu().numpy()
    for i, n in enumerate(rc.MODELZOO_FRAMES):
        assert np.array_equal(out[i:i + 1], g[n + "_u8"]), n


def test_detect_frames_known_answers_in_source_pixels(golden_dir):
    """test.py:34-68 on the raw bundled frames: person .87, bicycle .46, person .32 on 000139, nine cars on 000004, with the
    corners scaled to the frame by test.py's float64 arithmetic."""
    import model.detector as det
    import utils.utils as uu
    from utils import frames as uf
    frames = np.load(os.path.join(golden_dir, "frames_modelzoo.npz"))
    g = np.load(os.path.join(golden_dir, "images_modelzoo.npz"))
    w = synth.load_modelzoo_weights(golden_dir)
    m = det.Detector(80, 3, True)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
    m = m.cuda().eval()
    cfg = synth.coco_cfg()
    raw = [frames[n] for n in rc.MODELZOO_FRAMES]
    got = uf.detect_frames(m, raw, cfg, conf_thres=0.3, iou_thres=0.4)
    # the same batch from the stored network inputs through forward + fused decode/NMS, then test.py:57-68 line by line
    x = torch.from_numpy(np.concatenate([g[n + "_u8"] for n in rc.MODELZOO_FRAMES])).cuda()
    with torch.no_grad():
        want = uu.detect(m(x), cfg, 0.3, 0.4)
    for i, n in enumerate(rc.MODELZOO_FRAMES):
        h, w_, _ = raw[i].shape
        scale_h, scale_w = h / cfg["height"], w_ / cfg["width"]
        rows = got[i]
        assert rows.dtype == torch.float64 and rows.shape == want[i].shape
        corners = uf.int_corners(rows).tolist()
        for r, c, box in zip(rows.tolist(), corners, want[i].tolist()):
            assert r == [box[0] * scale_w, box[1] * scale_h, box[2] * scale_w, box[3] * scale_h, box[4], box[5]]
            assert c == [int(box[0] * scale_w), int(box[1] * scale_h), int(box[2] * scale_w), int(box[3] * scale_h)]
        ref = g[n + "_nms_0.3_0.4_rows"].astype(np.float64)           # the reference's rows at the network input size
        ref[:, [0, 2]] *= scale_w
        ref[:, [1, 3]] *= scale_h
        assert np.array_equal(rows.numpy()[:, 5], ref[:, 5])
        np.testing.assert_allclose(rows.numpy(), ref, rtol=1e-4, atol=2e-3 * max(scale_w, scale_h))
    assert [(int(r[5]), "%.2f" % r[4]) for r in got[0].tolist()] == [(0, "0.87"), (1, "0.46"), (0, "0.32")]
    assert ["%.2f" % r[4] for r in got[1].tolist()] == ["0.87", "0.85", "0.76", "0.75", "0.68", "0.60", "0.56", "0.47", "0.33"]
    assert all(int(r[5]) == 2 for r in got[1].tolist())


def test_fullhd_batch_of_64_equals_oracle():
    frames = np.random.default_rng(11).integers(0, 256, (64, 1080, 1920, 3), dtype=np.uint8)
    out = eng.resize_bgr(list(torch.from_numpy(frames).cuda()), 352, 352).cpu().numpy()
    for i in range(64):
        assert np.array_equal(out[i], ore.resize_bgr_planar(frames[i], 352, 352)), i

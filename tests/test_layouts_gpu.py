"""RGB, BGRA / RGBA, grey, planar RGB and packed YUV 4:2:2 frames on the device (resize_frames through yfv2_resize_strided_u8 and
yfv2_resize_yuv422_u8) against the frozen cv2.cvtColor + cv2.resize outputs and the numpy oracle, bit for bit, for every layout,
frame form and batch shape, batches mixing all 13 layouts, and detect_frames on every layout of the bundled images."""
import hashlib
import os

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import layout_cases as lc
import layout_oracle as lo
import synth
import yfv2_engine as eng
import yuv_cases as yc

pytestmark = pytest.mark.gpu


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def hwc(planar):
    return planar.permute(1, 2, 0).contiguous().cpu().numpy()


def device_view(a):
    """A numpy view on the device with the same strides and offset, inside a device copy of the array it views."""
    base = a if a.base is None else a.base
    d = torch.from_numpy(np.ascontiguousarray(base)).cuda()
    off = a.__array_interface__["data"][0] - base.__array_interface__["data"][0]
    return torch.as_strided(d, a.shape, a.strides, off)


def pitched(a, layout):
    """The frame copied into the middle of a larger device surface: rows (and planes) further apart, an offset of one row and two
    pixels (a whole 4:2:2 macropixel)."""
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    if layout == "rgb_chw":
        s = torch.zeros((4, a.shape[1] + 3, a.shape[2] + 6), dtype=torch.uint8, device="cuda")
        s[1:, 1:1 + a.shape[1], 2:2 + a.shape[2]] = t
        return s[1:, 1:1 + a.shape[1], 2:2 + a.shape[2]]
    s = torch.zeros((a.shape[0] + 3, a.shape[1] + 6) + a.shape[2:], dtype=torch.uint8, device="cuda")
    s[1:1 + a.shape[0], 2:2 + a.shape[1]] = t
    return s[1:1 + a.shape[0], 2:2 + a.shape[1]]


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "layout_cases.npz"))


@pytest.mark.parametrize("case", lc.CASES, ids=[c[0] for c in lc.CASES])
def test_bit_exact_against_cv2_golden(golden, case):
    name, layout, _, _, (H, W), _ = case
    out = eng.resize_frames([device_view(lc.case_input(case))], W, H, layout)
    assert out.shape == (1, 3, H, W) and out.dtype == torch.uint8
    got = hwc(out[0])
    if name + "_out" in golden:
        assert np.array_equal(got, golden[name + "_out"])
    assert np.array_equal(sha(got), golden[name + "_sha256"])


@pytest.mark.parametrize("case", lc.CASES, ids=[c[0] for c in lc.CASES])
def test_every_frame_form_gives_the_same_bytes(case):
    name, layout, _, _, (H, W), _ = case
    frame = lc.case_input(case)
    forms = {
        "host array": frame,
        "host contiguous array": np.ascontiguousarray(frame),
        "device contiguous tensor": torch.from_numpy(np.ascontiguousarray(frame)).cuda(),
        "device view of the case's surface": device_view(frame),
        "device pitched view": pitched(frame, layout),
    }
    want = eng.resize_frames([frame], W, H, layout)
    assert np.array_equal(want[0].cpu().numpy(), lo.resize_planar(frame, layout, W, H)), name
    for form, f in forms.items():
        assert torch.equal(eng.resize_frames([f], W, H, layout), want), (name, form)


def all_layout_frames():
    """One frame of each of the 13 layouts, of different sizes, ordered so that consecutive frames alternate descriptor kinds."""
    pick = {c[1]: c for c in lc.CASES if c[0].endswith("_odd")}
    pick["rgb_chw"] = next(c for c in lc.CASES if c[0] == "rgb_chw_chw_every_other")
    pick["yvyu"] = next(c for c in lc.CASES if c[0] == "yvyu_crop")
    frames = {k: device_view(lc.case_input(c)) for k, c in pick.items()}
    for c in yc.CASES[:5]:                                     # nv12, nv12, i420, nv21, yv12 single buffers
        frames.setdefault(c[1], torch.from_numpy(yc.case_input(c)).cuda())
    frames["bgr"] = torch.from_numpy(np.random.RandomState(5).randint(0, 256, (211, 157, 3)).astype(np.uint8)).cuda()
    order = ["bgr", "rgb", "nv12", "yuyv", "bgra", "i420", "uyvy", "rgba", "gray", "nv21", "rgb_chw", "yvyu", "yv12"]
    assert sorted(order) == sorted(eng.LAYOUTS)
    return [frames[k] for k in order], order


def oracle(frame, layout, W, H):
    if isinstance(frame, torch.Tensor):
        frame = frame.cpu().numpy()
    return lo.resize_planar(frame, layout, W, H)


@pytest.mark.parametrize("H,W", [(352, 352), (96, 160)])
def test_batch_mixing_all_13_layouts(H, W):
    frames, layouts = all_layout_frames()
    batch = eng.resize_frames(frames, W, H, layouts)
    for i, (f, layout) in enumerate(zip(frames, layouts)):
        assert torch.equal(batch[i], eng.resize_frames([f], W, H, layout)[0]), layout
        assert np.array_equal(batch[i].cpu().numpy(), oracle(f, layout, W, H)), layout
    # the same frames into a caller's buffer, and the runs of one kind in a different order
    out = torch.full((len(frames), 3, H, W), 7, dtype=torch.uint8, device="cuda")
    assert eng.resize_frames(frames, W, H, layouts, out=out) is out and torch.equal(out, batch)
    perm = sorted(range(len(frames)), key=lambda i: eng._KIND[layouts[i]])
    again = eng.resize_frames([frames[i] for i in perm], W, H, [layouts[i] for i in perm])
    assert torch.equal(again, batch[perm])


def random_frame(rs, layout):
    h, w = rs.randint(1, 90), 2 * rs.randint(1, 45)
    if layout in ("nv12", "nv21", "i420", "yv12"):
        return rs.randint(0, 256, (2 * (h // 2 + 1) * 3 // 2, w)).astype(np.uint8)
    if layout == "bgr":
        return rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
    return rs.randint(0, 256, lc.frame_shape(layout, h, w)).astype(np.uint8)


def test_300_frames_span_several_launches_of_each_kind():
    """120 strided frames (two launches of 80 descriptors), 120 packed 4:2:2 frames (two launches of 96), then 60 frames of random
    layouts (many short runs of every kind), all of random sizes, in one call."""
    rs = np.random.RandomState(17)
    layouts = ([lc.LAYOUTS[rs.randint(5)] for _ in range(120)] + [lc.YUV422[rs.randint(3)] for _ in range(120)]
               + [eng.LAYOUTS[rs.randint(13)] for _ in range(60)])
    frames = [random_frame(rs, lay) for lay in layouts]
    out = eng.resize_frames(frames, 37, 29, layouts).cpu().numpy()
    for i, (f, layout) in enumerate(zip(frames, layouts)):
        assert np.array_equal(out[i], oracle(f, layout, 37, 29)), (i, layout)


@pytest.mark.parametrize("layouts", [("rgb", "bgra", "rgba", "gray", "rgb_chw"), ("yuyv", "uyvy", "yvyu")])
def test_fullhd_batch_of_64_per_descriptor_kind_equals_oracle(layouts):
    rng = np.random.default_rng(19)
    names = [layouts[i % len(layouts)] for i in range(64)]
    frames = [torch.from_numpy(rng.integers(0, 256, lc.frame_shape(n, 1080, 1920), dtype=np.uint8)).cuda() for n in names]
    out = eng.resize_frames(frames, 352, 352, names).cpu().numpy()
    for i, (f, n) in enumerate(zip(frames, names)):
        assert np.array_equal(out[i], oracle(f, n, 352, 352)), (i, n)


def bundled(golden, golden_dir, img, layout):
    return lc.bundled(golden, np.load(os.path.join(golden_dir, "frames_modelzoo.npz")), img, layout)


def modelzoo_detector(golden_dir):
    import model.detector as det
    w = synth.load_modelzoo_weights(golden_dir)
    m = det.Detector(80, 3, True)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
    return m.cuda().eval()


@pytest.mark.parametrize("layout", ["rgb", "bgra", "rgba", "rgb_chw"])
def test_lossless_layouts_of_the_bundled_images_give_the_bgr_answers(golden, golden_dir, layout):
    """The network inputs are the stored ones of the BGR frames, and detect_frames returns exactly the BGR rows: person .87,
    bicycle .46, person .32 on 000139 and nine cars on 000004, in pixels of each frame."""
    from utils import frames as uf
    images = np.load(os.path.join(golden_dir, "images_modelzoo.npz"))
    raw = [torch.from_numpy(bundled(golden, golden_dir, n, layout)).cuda() for n in lc.MODELZOO_FRAMES]
    x = eng.resize_frames(raw, 352, 352, layout).cpu().numpy()
    for i, n in enumerate(lc.MODELZOO_FRAMES):
        assert np.array_equal(x[i:i + 1], images[n + "_u8"]), n
    m = modelzoo_detector(golden_dir)
    cfg = synth.coco_cfg()
    bgr = np.load(os.path.join(golden_dir, "frames_modelzoo.npz"))
    want = uf.detect_frames(m, [bgr[n] for n in lc.MODELZOO_FRAMES], cfg, conf_thres=0.3, iou_thres=0.4, layout="bgr")
    got = uf.detect_frames(m, raw, cfg, conf_thres=0.3, iou_thres=0.4, layout=layout)
    for a, b in zip(got, want):
        assert a.dtype == torch.float64 and torch.equal(a, b)
    assert [(int(r[5]), "%.2f" % r[4]) for r in got[0].tolist()] == [(0, "0.87"), (1, "0.46"), (0, "0.32")]
    assert ["%.2f" % r[4] for r in got[1].tolist()] == ["0.87", "0.85", "0.76", "0.75", "0.68", "0.60", "0.56", "0.47", "0.33"]
    # one call mixing this layout with BGR frames gives the same rows per frame
    mixed = uf.detect_frames(m, [raw[0], bgr[lc.MODELZOO_FRAMES[1]]], cfg, conf_thres=0.3, iou_thres=0.4, layout=[layout, "bgr"])
    assert torch.equal(mixed[0], want[0]) and torch.equal(mixed[1], want[1])


@pytest.mark.parametrize("layout", ["gray", "yuyv", "uyvy", "yvyu"])
def test_detect_frames_on_lossy_layouts_in_source_pixels(golden, golden_dir, layout):
    """test.py:34-68 on the bundled images delivered as grey or 4:2:2: detect_frames(layout=...) gives, bit for bit, the rows of
    forward + detect on cv2's 352 x 352 BGR resize of the same converted frame, scaled back by test.py's float64 arithmetic."""
    import utils.utils as uu
    from utils import frames as uf
    m = modelzoo_detector(golden_dir)
    cfg = synth.coco_cfg()
    raw = [bundled(golden, golden_dir, n, layout) for n in lc.MODELZOO_FRAMES]
    got = uf.detect_frames(m, raw, cfg, conf_thres=0.3, iou_thres=0.4, layout=layout)
    # cv2's 352 x 352 BGR resize of each converted frame: the oracle's bytes, which the golden file pins to cv2's by SHA-256
    x = np.stack([lo.resize_planar(f, layout, 352, 352) for f in raw])
    for n, xi in zip(lc.MODELZOO_FRAMES, x):
        assert np.array_equal(sha(xi.transpose(1, 2, 0)), golden["%s_%s_bgr352_sha256" % (n, layout)]), n
    x = torch.from_numpy(x).cuda()
    with torch.no_grad():
        want = uu.detect(m(x), cfg, 0.3, 0.4)
    for i, f in enumerate(raw):
        h, w_ = f.shape[:2]
        scale_h, scale_w = h / cfg["height"], w_ / cfg["width"]
        rows = got[i]
        assert rows.dtype == torch.float64 and rows.shape == want[i].shape and rows.shape[0] > 0
        for r, c, box in zip(rows.tolist(), uf.int_corners(rows).tolist(), want[i].tolist()):
            assert r == [box[0] * scale_w, box[1] * scale_h, box[2] * scale_w, box[3] * scale_h, box[4], box[5]]
            assert c == [int(box[0] * scale_w), int(box[1] * scale_h), int(box[2] * scale_w), int(box[3] * scale_h)]
    print("detect_frames(layout=%r): %s" % (layout, [[(int(r[5]), "%.3f" % r[4]) for r in g.tolist()] for g in got]))

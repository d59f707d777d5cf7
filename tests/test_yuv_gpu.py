"""YUV 4:2:0 frames on the device (yfv2_resize_yuv420_u8 through the C ABI) against the frozen cv2.cvtColor + cv2.resize outputs
and the numpy oracle, bit for bit, for every layout, frame form and batch shape; and detect_frames on YUV frames."""
import hashlib
import os

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import resize_cases as rc
import synth
import yfv2_engine as eng
import yuv_cases as yc
import yuv_oracle as yo

pytestmark = pytest.mark.gpu


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def hwc(planar):
    return planar.permute(1, 2, 0).contiguous().cpu().numpy()


def on_device(frame):
    """A case's frame on the device in the same form: a single buffer, or plane views with the pitches and offsets of the numpy
    views, into one device copy of each surface (an NV12 / NV21 surface keeps luma and chroma in one allocation)."""
    if not isinstance(frame, tuple):
        return torch.from_numpy(frame).cuda()
    surfaces, views = {}, []
    for p in frame:
        base = p.base
        if id(base) not in surfaces:
            surfaces[id(base)] = torch.from_numpy(base).cuda()
        d = surfaces[id(base)]
        off = p.__array_interface__["data"][0] - base.__array_interface__["data"][0]
        views.append(torch.as_strided(d, p.shape, p.strides, off))
    return tuple(views)


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "yuv_cases.npz"))


@pytest.mark.parametrize("case", yc.CASES, ids=[c[0] for c in yc.CASES])
def test_bit_exact_against_cv2_golden(golden, case):
    name, layout, _, _, (H, W), _ = case
    frame = on_device(yc.case_input(case))
    out = eng.resize_yuv420([frame], W, H, layout)
    assert out.shape == (1, 3, H, W) and out.dtype == torch.uint8
    got = hwc(out[0])
    if name + "_out" in golden:
        assert np.array_equal(got, golden[name + "_out"])
    assert np.array_equal(sha(got), golden[name + "_sha256"])


def test_whole_colour_cube_is_bit_exact(golden):
    """Every (y, u, v) triple, NV12 at identity size, in one launch of 64 frames."""
    frames = [torch.from_numpy(yc.cube_frame(k)).cuda() for k in range(yc.CUBE_FRAMES)]
    out = eng.resize_yuv420(frames, 512, 512, "nv12")
    for k in range(yc.CUBE_FRAMES):
        assert np.array_equal(sha(hwc(out[k])), golden["cube_%02d_sha256" % k]), k


def test_bundled_images_give_cv2s_result(golden):
    for name in yc.MODELZOO_FRAMES:
        i420 = golden[name + "_i420"]
        want = golden[name + "_bgr352"]
        for buf, layout in ((i420, "i420"), (yc.i420_to_nv12(i420), "nv12")):
            assert np.array_equal(hwc(eng.resize_yuv420([buf], 352, 352, layout)[0]), want), (name, layout)


@pytest.mark.parametrize("case", [c for c in yc.CASES if c[5] is not None], ids=[c[0] for c in yc.CASES if c[5] is not None])
def test_single_buffer_planes_and_pitched_surface_agree(case):
    name, layout, _, _, (H, W), _ = case
    views = yc.case_input(case)
    forms = {
        "device pitched views": on_device(views),
        "host pitched views": views,
        "device contiguous planes": tuple(torch.from_numpy(np.ascontiguousarray(p)).cuda() for p in views),
        "device single buffer": torch.from_numpy(yc.single_buffer(views, layout)).cuda(),
        "host single buffer": yc.single_buffer(views, layout),
    }
    want = eng.resize_yuv420([forms["device pitched views"]], W, H, layout)
    assert np.array_equal(want[0].cpu().numpy(), yo.resize_frame_planar(views, layout, W, H))
    for form, f in forms.items():
        assert torch.equal(eng.resize_yuv420([f], W, H, layout), want), (name, form)


def test_even_offset_crops_of_a_pitched_surface_equal_contiguous_copies():
    rs = np.random.RandomState(31)
    surf = torch.from_numpy(rs.randint(0, 256, (1088 + 544, 2048)).astype(np.uint8)).cuda()
    for (y0, x0, h, w) in [(0, 0, 1080, 1920), (2, 2, 1078, 1918), (130, 6, 516, 770), (1078, 0, 2, 2048), (0, 2044, 1088, 4)]:
        y, uv = surf[y0:y0 + h, x0:x0 + w], surf[1088 + y0 // 2:1088 + (y0 + h) // 2, x0:x0 + w]
        for layout in ("nv12", "nv21"):
            a = eng.resize_yuv420([(y, uv)], 352, 352, layout)
            b = eng.resize_yuv420([(y.contiguous(), uv.contiguous())], 352, 352, layout)
            assert torch.equal(a, b), (y0, x0, h, w, layout)
            assert np.array_equal(a[0].cpu().numpy(), yo.resize_frame_planar((y.cpu().numpy(), uv.cpu().numpy()), layout, 352, 352))


@pytest.mark.parametrize("H,W", [(352, 352), (96, 160)])
def test_batch_mixing_sizes_and_all_four_layouts(H, W):
    frames = [on_device(yc.case_input(c)) for c in yc.CASES]
    layouts = [c[1] for c in yc.CASES]
    assert set(layouts) == set(yo.LAYOUTS)
    batch = eng.resize_yuv420(frames, W, H, layouts)
    for i, (f, layout) in enumerate(zip(frames, layouts)):
        assert torch.equal(batch[i], eng.resize_yuv420([f], W, H, layout)[0]), yc.CASES[i][0]
        assert np.array_equal(batch[i].cpu().numpy(), yo.resize_frame_planar(yc.case_input(yc.CASES[i]), layout, W, H)), yc.CASES[i][0]


def test_many_frames_span_several_launches():
    """300 frames of random even sizes and layouts: more than four launches of 64 descriptors, every frame in its own slot."""
    rs = np.random.RandomState(12)
    frames, layouts = [], []
    for _ in range(300):
        h, w = 2 * rs.randint(1, 45), 2 * rs.randint(1, 45)
        frames.append(rs.randint(0, 256, (h * 3 // 2, w)).astype(np.uint8))
        layouts.append(yo.LAYOUTS[rs.randint(4)])
    out = eng.resize_yuv420(frames, 37, 29, layouts).cpu().numpy()
    for i, (f, layout) in enumerate(zip(frames, layouts)):
        assert np.array_equal(out[i], yo.resize_frame_planar(f, layout, 37, 29)), i


def test_fullhd_nv12_batch_of_64_equals_oracle():
    frames = np.random.default_rng(13).integers(0, 256, (64, 1620, 1920), dtype=np.uint8)
    out = eng.resize_yuv420(list(torch.from_numpy(frames).cuda()), 352, 352, "nv12").cpu().numpy()
    for i in range(64):
        assert np.array_equal(out[i], yo.resize_frame_planar(frames[i], "nv12", 352, 352)), i


@pytest.mark.parametrize("layout", ["i420", "nv12"])
def test_detect_frames_on_yuv_frames_in_source_pixels(golden_dir, golden, layout):
    """test.py:34-68 on the bundled images delivered as YUV: detect_frames(layout=...) gives, bit for bit, the rows of forward +
    detect on cv2's 352 x 352 BGR resize of the same YUV frame, scaled back to the frame by test.py's float64 arithmetic."""
    import model.detector as det
    import utils.utils as uu
    from utils import frames as uf
    w = synth.load_modelzoo_weights(golden_dir)
    m = det.Detector(80, 3, True)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
    m = m.cuda().eval()
    cfg = synth.coco_cfg()
    raw = [golden[n + "_i420"] for n in yc.MODELZOO_FRAMES]
    if layout == "nv12":
        raw = [yc.i420_to_nv12(f) for f in raw]
    got = uf.detect_frames(m, raw, cfg, conf_thres=0.3, iou_thres=0.4, layout=layout)
    x = torch.from_numpy(np.stack([golden[n + "_bgr352"].transpose(2, 0, 1) for n in yc.MODELZOO_FRAMES])).cuda()
    with torch.no_grad():
        want = uu.detect(m(x), cfg, 0.3, 0.4)
    frames = np.load(os.path.join(golden_dir, "frames_modelzoo.npz"))
    for i, n in enumerate(rc.MODELZOO_FRAMES):
        h, w_ = frames[n].shape[:2]
        scale_h, scale_w = h / cfg["height"], w_ / cfg["width"]
        rows = got[i]
        assert rows.dtype == torch.float64 and rows.shape == want[i].shape and rows.shape[0] > 0
        for r, c, box in zip(rows.tolist(), uf.int_corners(rows).tolist(), want[i].tolist()):
            assert r == [box[0] * scale_w, box[1] * scale_h, box[2] * scale_w, box[3] * scale_h, box[4], box[5]]
            assert c == [int(box[0] * scale_w), int(box[1] * scale_h), int(box[2] * scale_w), int(box[3] * scale_h)]
    print("detect_frames(layout=%r): %s" % (layout, [[(int(r[5]), "%.3f" % r[4]) for r in g.tolist()] for g in got]))

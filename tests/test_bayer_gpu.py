"""Raw Bayer frames on the device (resize_frames through yfv2_resize_bayer_u8, encode_jpeg through YFV2_JPEG_SRC_BAYER) against the
frozen cv2.cvtColor(COLOR_Bayer??2BGR / _EA) + crop + cv2.resize / cv2.imencode outputs and the numpy oracle, bit for bit: every
case and frame form, windows, batches mixing the 8 Bayer layouts with the other 13 and spanning several launches, and
detect_frames, detect_tiled, track_frames and encode_detections on Bayer mosaics of the bundled images."""
import hashlib
import os

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import bayer_cases as bc
import bayer_oracle as bo
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


def pitched(a):
    """The raw frame copied into the middle of a larger device surface: rows further apart, an offset of one row and 3 bytes."""
    s = torch.zeros((a.shape[0] + 3, a.shape[1] + 9), dtype=torch.uint8, device="cuda")
    s[1:1 + a.shape[0], 3:3 + a.shape[1]] = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return s[1:1 + a.shape[0], 3:3 + a.shape[1]]


def as_frame(raw, layout, window):
    """What resize_frames takes for a case: the raw frame, or the BayerWindow crop_frame makes of it."""
    return raw if window is None else eng.crop_frame(raw, layout, *window)


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "bayer_cases.npz"))


@pytest.mark.parametrize("case", bc.CASES, ids=[c[0] for c in bc.CASES])
def test_bit_exact_against_cv2_golden_and_oracle(golden, case):
    name, layout, _, _, (H, W), window, _ = case
    raw = bc.case_input(case)
    out = eng.resize_frames([as_frame(device_view(raw), layout, window)], W, H, layout)
    assert out.shape == (1, 3, H, W) and out.dtype == torch.uint8
    got = hwc(out[0])
    if name + "_out" in golden:
        assert np.array_equal(got, golden[name + "_out"])
    assert np.array_equal(sha(got), golden[name + "_sha256"])
    assert np.array_equal(out[0].cpu().numpy(), bo.resize_planar(raw, layout, W, H, bc.window_of(case)))


@pytest.mark.parametrize("case", bc.CASES[::3], ids=[c[0] for c in bc.CASES[::3]])
def test_every_frame_form_gives_the_same_bytes(case):
    name, layout, _, _, (H, W), window, _ = case
    raw = bc.case_input(case)
    want = eng.resize_frames([as_frame(raw, layout, window)], W, H, layout)
    forms = {
        "host contiguous array": np.ascontiguousarray(raw),
        "device contiguous tensor": torch.from_numpy(np.ascontiguousarray(raw)).cuda(),
        "device view of the case's surface": device_view(raw),
        "device pitched view": pitched(raw),
        "device column-strided view (copied)": torch.from_numpy(np.ascontiguousarray(raw).T.copy()).cuda().T,
    }
    for form, f in forms.items():
        assert torch.equal(eng.resize_frames([as_frame(f, layout, window)], W, H, layout), want), (name, form)
    if window is not None:                       # the window given directly, not through crop_frame
        assert torch.equal(eng.resize_frames([eng.BayerWindow(pitched(raw), *window)], W, H, layout), want), name


def other_layout_frames():
    """One frame of each of the 13 other layouts, as test_layouts_gpu.py builds them."""
    pick = {c[1]: c for c in lc.CASES if c[0].endswith("_odd")}
    frames = {k: torch.from_numpy(np.ascontiguousarray(lc.case_input(c))).cuda() for k, c in pick.items()}
    for c in yc.CASES[:5]:
        frames.setdefault(c[1], torch.from_numpy(yc.case_input(c)).cuda())
    frames["bgr"] = torch.from_numpy(np.random.RandomState(5).randint(0, 256, (211, 157, 3)).astype(np.uint8)).cuda()
    assert sorted(frames) == sorted(eng.LAYOUTS)
    return frames


def bayer_frame(rs, layout):
    """A random raw frame of random size, pitched on the device, whole or as a random window."""
    fh, fw = rs.randint(1, 70), rs.randint(1, 90)
    raw = pitched(rs.randint(0, 256, (fh, fw)).astype(np.uint8))
    if rs.randint(2):
        return raw
    w, h = rs.randint(1, fw + 1), rs.randint(1, fh + 1)
    return eng.crop_frame(raw, layout, rs.randint(0, fw - w + 1), rs.randint(0, fh - h + 1), w, h)


def oracle(frame, layout, W, H):
    if isinstance(frame, eng.BayerWindow):
        return bo.resize_planar(frame.raw.cpu().numpy(), layout, W, H, (frame.x0, frame.y0, frame.w, frame.h))
    if layout in eng.BAYER_LAYOUTS:
        return bo.resize_planar(frame.cpu().numpy(), layout, W, H)
    return lo.resize_planar(frame.cpu().numpy(), layout, W, H)


@pytest.mark.parametrize("H,W", [(352, 352), (96, 160)])
def test_batch_mixing_all_8_bayer_layouts_with_the_other_13(H, W):
    rs = np.random.RandomState(23)
    others = other_layout_frames()
    order = ["bgr", "bayer_bg", "rgb", "bayer_gb_ea", "bayer_rg", "nv12", "yuyv", "bayer_gr", "bayer_bg_ea", "bgra", "i420",
             "bayer_gb", "uyvy", "rgba", "bayer_rg_ea", "gray", "nv21", "bayer_gr_ea", "rgb_chw", "yvyu", "yv12"]
    assert sorted(order) == sorted(eng.LAYOUTS + eng.BAYER_LAYOUTS)
    frames = [bayer_frame(rs, lay) if lay in eng.BAYER_LAYOUTS else others[lay] for lay in order]
    batch = eng.resize_frames(frames, W, H, order)
    for i, (f, layout) in enumerate(zip(frames, order)):
        assert torch.equal(batch[i], eng.resize_frames([f], W, H, layout)[0]), layout
        assert np.array_equal(batch[i].cpu().numpy(), oracle(f, layout, W, H)), layout


def test_more_than_one_launch_of_bayer_frames():
    """150 Bayer frames (three launches of at most 64 descriptors) of random sizes, layouts, windows and pitches in one call, then
    the same with frames of other layouts between them."""
    rs = np.random.RandomState(29)
    layouts = [eng.BAYER_LAYOUTS[rs.randint(8)] for _ in range(150)]
    frames = [bayer_frame(rs, lay) for lay in layouts]
    out = eng.resize_frames(frames, 37, 29, layouts)
    for i, (f, layout) in enumerate(zip(frames, layouts)):
        assert np.array_equal(out[i].cpu().numpy(), oracle(f, layout, 37, 29)), (i, layout)
    bgr = torch.from_numpy(rs.randint(0, 256, (33, 45, 3)).astype(np.uint8)).cuda()
    mixed_f, mixed_l = frames[:70] + [bgr] + frames[70:], layouts[:70] + ["bgr"] + layouts[70:]
    mixed = eng.resize_frames(mixed_f, 37, 29, mixed_l)
    assert torch.equal(mixed[:70], out[:70]) and torch.equal(mixed[71:], out[70:])


def test_windows_equal_the_crop_of_the_converted_frame():
    """crop_frame windows of every layout, odd offsets, edges and 1-pixel sizes included, and crops of crops: the oracle of
    cv2.cvtColor(raw)[window], resized (an identity resize shows the window's converted pixels themselves)."""
    rs = np.random.RandomState(31)
    raw = rs.randint(0, 256, (121, 161)).astype(np.uint8)
    d = pitched(raw)
    for layout in eng.BAYER_LAYOUTS:
        whole = bo.to_bgr(raw, layout)
        for x0, y0, w, h in [(0, 0, 161, 121), (0, 0, 1, 1), (160, 120, 1, 1), (37, 21, 55, 43), (1, 1, 159, 119),
                             (0, 60, 161, 1), (80, 0, 1, 121), (158, 117, 3, 4)]:
            for f in (raw, d):
                win = eng.crop_frame(f, layout, x0, y0, w, h)
                got = hwc(eng.resize_frames([win], w, h, layout)[0])
                assert np.array_equal(got, whole[y0:y0 + h, x0:x0 + w]), (layout, (x0, y0, w, h))
        inner = eng.crop_frame(eng.crop_frame(d, layout, 11, 7, 120, 90), layout, 5, 3, 101, 71)
        got = hwc(eng.resize_frames([inner], 101, 71, layout)[0])
        assert np.array_equal(got, whole[10:81, 16:117]), layout
        assert not np.array_equal(got, bo.to_bgr(raw[10:81, 16:117], layout))       # a crop of the raw bytes would differ


def test_frames_under_3_pixels_on_a_side_give_zeros():
    rs = np.random.RandomState(37)
    for fh, fw in [(1, 1), (1, 200), (200, 1), (2, 2), (2, 177), (177, 2)]:
        raw = rs.randint(1, 256, (fh, fw)).astype(np.uint8)
        for layout in eng.BAYER_LAYOUTS:
            out = eng.resize_frames([raw, eng.crop_frame(raw, layout, 0, 0, 1, 1)], 40, 30, layout)
            assert not out.any(), (fh, fw, layout)


@pytest.mark.parametrize("c", bc.ENCODE_CASES, ids=[c["name"] for c in bc.ENCODE_CASES])
def test_encode_jpeg_byte_identical_to_cv2(golden, c):
    raw = pitched(bc.raw_frame(c["seed"], c["fh"], c["fw"]))
    frame = raw if c["window"] is None else eng.crop_frame(raw, c["layout"], *c["window"])
    regions = None if c["region"] is None else [(0,) + tuple(c["region"])]
    got = eng.encode_jpeg([frame], c["quality"], c["sampling"], layout=c["layout"], regions=regions)[0]
    if c["name"] + ".jpg" in golden:
        assert got == golden[c["name"] + ".jpg"].tobytes()
    else:
        assert len(got) == int(golden[c["name"] + ".len"])
        assert hashlib.sha256(got).digest() == golden[c["name"] + ".sha"].tobytes()


def test_encode_jpeg_of_bayer_is_the_encode_of_the_oracle_bgr():
    """Whole frames, windows and regions of several Bayer layouts in one call with BGR frames: each output equals the encode of
    the oracle's converted frame (the BGR path), one output per region."""
    rs = np.random.RandomState(41)
    raws = [rs.randint(0, 256, (97 + k, 131 + 2 * k)).astype(np.uint8) for k in range(4)]
    lays = ["bayer_bg", "bayer_gr_ea", "bayer_rg", "bayer_gb_ea"]
    frames = [raws[0], eng.crop_frame(raws[1], lays[1], 3, 5, 101, 77), pitched(raws[2]), raws[3]]
    bgrs = [bo.to_bgr(raws[0], lays[0]), bo.window_bgr(raws[1], lays[1], 3, 5, 101, 77), bo.to_bgr(raws[2], lays[2]),
            bo.to_bgr(raws[3], lays[3])]
    regions = [(0, 0, 0, 131, 97), (1, 0, 0, 101, 77), (1, 17, 9, 33, 41), (2, 100, 50, 33, 49), (3, 1, 1, 9, 9)]
    got = eng.encode_jpeg(frames + bgrs, 90, "444", layout=lays + ["bgr"] * 4,
                          regions=regions + [(r[0] + 4,) + r[1:] for r in regions])
    assert got[:5] == got[5:]


def mosaics(golden_dir):
    """The bundled images as raw frames of each pattern (each pixel keeps its site's channel), and the oracle's demosaic of each."""
    bgr = np.load(os.path.join(golden_dir, "frames_modelzoo.npz"))
    return [(n, lay, bo.mosaic(bgr[n], lay)) for n in lc.MODELZOO_FRAMES for lay in eng.BAYER_LAYOUTS]


def modelzoo_detector(golden_dir):
    import model.detector as det
    w = synth.load_modelzoo_weights(golden_dir)
    m = det.Detector(80, 3, True)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
    return m.cuda().eval()


def test_detect_frames_and_tiled_on_mosaics_equal_the_oracle_bgr(golden_dir):
    from utils import frames as uf
    m, cfg = modelzoo_detector(golden_dir), synth.coco_cfg()
    cases = mosaics(golden_dir)
    raws, lays = [r for _, _, r in cases], [lay for _, lay, _ in cases]
    bgrs = [np.ascontiguousarray(bo.to_bgr(r, lay)) for r, lay in zip(raws, lays)]
    got = uf.detect_frames(m, raws, cfg, conf_thres=0.3, iou_thres=0.4, layout=lays)
    want = uf.detect_frames(m, bgrs, cfg, conf_thres=0.3, iou_thres=0.4, layout="bgr")
    for (n, lay, _), a, b in zip(cases, got, want):
        assert a.dtype == torch.float64 and torch.equal(a, b), (n, lay)
    assert sum(g.shape[0] for g in got) > 0
    # one call mixing Bayer frames with the BGR frames
    mixed = uf.detect_frames(m, [raws[0], bgrs[9], raws[15]], cfg, conf_thres=0.3, iou_thres=0.4,
                             layout=[lays[0], "bgr", lays[15]])
    assert all(torch.equal(a, want[k]) for a, k in zip(mixed, (0, 9, 15)))
    # tiles: windows of the converted frame, odd origins and sizes included
    pick = [0, 5, 10, 15]
    tiled = uf.detect_tiled(m, [torch.from_numpy(raws[k]).cuda() for k in pick], cfg, 3, 2, 0.2, True,
                            layout=[lays[k] for k in pick], conf_thres=0.2)
    tiled_bgr = uf.detect_tiled(m, [bgrs[k] for k in pick], cfg, 3, 2, 0.2, True, layout="bgr", conf_thres=0.2)
    for a, b in zip(tiled, tiled_bgr):
        assert a.dtype == torch.float64 and torch.equal(a, b)
    assert sum(a.shape[0] for a in tiled) > 0
    # detect_regions of a window, and encode_detections of the rows
    win = eng.crop_frame(raws[0], lays[0], 31, 17, 301, 251)
    regs = uf.detect_regions(m, [win], cfg, [[(0, 0, 301, 251), (7, 9, 151, 121)]], layout=lays[0], conf_thres=0.2)
    regs_bgr = uf.detect_regions(m, [np.ascontiguousarray(bgrs[0][17:268, 31:332])], cfg,
                                 [[(0, 0, 301, 251), (7, 9, 151, 121)]], layout="bgr", conf_thres=0.2)
    assert torch.equal(regs[0], regs_bgr[0])
    files = uf.encode_detections([raws[0], win], [got[0], regs[0]], layout=lays[0], quality=90)
    files_bgr = uf.encode_detections([bgrs[0], np.ascontiguousarray(bgrs[0][17:268, 31:332])], [got[0], regs[0]], quality=90)
    assert files == files_bgr and len(files[0]) == got[0].shape[0]


def test_track_frames_on_mosaics_equal_the_oracle_bgr(golden_dir):
    """A zoom and pan over the mosaic of 000139.jpg as Bayer windows in stream 0 and of 000004.jpg in stream 1, against the same
    calls on the oracle's converted windows, step by step."""
    from utils.tracking import track_frames
    m, cfg = modelzoo_detector(golden_dir), synth.coco_cfg()
    bgr = np.load(os.path.join(golden_dir, "frames_modelzoo.npz"))
    lays = ["bayer_gr_ea", "bayer_bg"]
    raws = [torch.from_numpy(bo.mosaic(bgr[n], lay)).cuda() for n, lay in zip(("000139", "000004"), lays)]
    convs = [bo.to_bgr(r.cpu().numpy(), lay) for r, lay in zip(raws, lays)]
    tracker, tracker_bgr = eng.Tracker("cuda", 2, 64), eng.Tracker("cuda", 2, 64)
    total = 0
    for k in range(6):
        frames, frames_bgr = [], []
        for r, c, lay in zip(raws, convs, lays):
            h, w = r.shape
            x0, y0 = 3 * k, 5 * k                    # odd offsets: windows of the converted frame
            frames.append(eng.crop_frame(r, lay, x0, y0, w - 2 * x0, h - y0 - k))
            frames_bgr.append(np.ascontiguousarray(c[y0:h - k, x0:w - x0]))
        got = track_frames(m, tracker, frames, cfg, layout=lays)
        want = track_frames(m, tracker_bgr, frames_bgr, cfg, layout="bgr")
        for a, b in zip(got, want):
            assert a.dtype == torch.float64 and torch.equal(a, b), k
        total += sum(a.shape[0] for a in got)
    assert total > 0

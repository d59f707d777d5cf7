"""Lens-corrected views on the device (resize_frames through yfv2_resize_remap_u8, remap_frames through yfv2_remap_u8) against the
frozen cv2.cvtColor + cv2.remap + crop + cv2.resize / cv2.imencode outputs and the numpy oracle, bit for bit: every case, frame
and map form, identity maps, batches mixing views with plain frames of every layout over several launches, and detect_frames,
detect_tiled, track_frames, encode_jpeg and encode_detections on undistorted views of the bundled images."""
import hashlib
import os

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import bayer_oracle as bo
import layout_cases as lc
import remap_cases as rc
import remap_oracle as ro
import synth
import yfv2_engine as eng
import yuv_cases as yc

pytestmark = pytest.mark.gpu


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def hwc(planar):
    return planar.permute(1, 2, 0).contiguous().cpu().numpy()


def pitched(a):
    """An array copied into the middle of a larger device surface: rows further apart and an offset (a 2-D or HWC frame)."""
    a = np.ascontiguousarray(a)
    s = torch.zeros((a.shape[0] + 3, a.shape[1] + 9) + a.shape[2:], dtype=torch.uint8, device="cuda")
    s[1:1 + a.shape[0], 3:3 + a.shape[1]] = torch.from_numpy(a).cuda()
    return s[1:1 + a.shape[0], 3:3 + a.shape[1]]


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "remap_cases.npz"))


def inner_frame(c, frame):
    """What the case's maps address, as the library takes it: the frame, or crop_frame's window of it."""
    return frame if c["inner"] is None else eng.crop_frame(frame, c["layout"], *c["inner"])


def case_view(c, golden, frame=None, maps=None):
    frame = torch.from_numpy(rc.case_frame(c)).cuda() if frame is None else frame
    maps = eng.RemapMaps(*rc.case_maps(c, golden)) if maps is None else maps
    return eng.RemapView(inner_frame(c, frame), maps, *rc.view_window(c))


def oracle_bgr(c, golden):
    img = ro.inner_bgr(rc.case_frame(c), c["layout"], c["inner"])
    return img, rc.fixed_maps(c, golden)


@pytest.mark.parametrize("c", rc.CASES, ids=[c["name"] for c in rc.CASES])
def test_bit_exact_against_cv2_golden_and_oracle(golden, c):
    name, (W, H) = c["name"], c["target"]
    view = case_view(c, golden)
    out = eng.resize_frames([view], W, H, c["layout"])
    assert out.shape == (1, 3, H, W) and out.dtype == torch.uint8
    got = hwc(out[0])
    if name + "_out" in golden:
        assert np.array_equal(got, golden[name + "_out"])
    assert np.array_equal(sha(got), golden[name + "_sha256"])
    img, (m1, m2) = oracle_bgr(c, golden)
    assert np.array_equal(out[0].cpu().numpy(), ro.resize_planar(img, m1, m2, rc.view_window(c), W, H))
    rem = eng.remap_frames([view], c["layout"])[0]
    assert rem.shape == (view.h, view.w, 3) and rem.dtype == torch.uint8 and rem.is_cuda
    rem = rem.cpu().numpy()
    if name + "_remap" in golden:
        assert np.array_equal(rem, golden[name + "_remap"])
    assert np.array_equal(sha(rem), golden[name + "_remap_sha256"])


@pytest.mark.parametrize("layout", ["bgr", "nv12", "i420", "gray", "rgb_chw", "yuyv", "bayer_gb_ea", "rgba"])
def test_integer_identity_map_gives_the_plain_resize(layout):
    fh, fw = 76, 98
    frame = torch.from_numpy(rc.frame(layout, 77, fh, fw)).cuda()
    v, u = np.meshgrid(np.arange(fh, dtype=np.float32), np.arange(fw, dtype=np.float32), indexing="ij")
    view = eng.RemapView(frame, eng.RemapMaps(u, v))
    for W, H in ((352, 352), (98, 76), (37, 29)):
        assert torch.equal(eng.resize_frames([view], W, H, layout), eng.resize_frames([frame], W, H, layout)), (layout, W, H)
    assert np.array_equal(eng.remap_frames([view], layout)[0].cpu().numpy(), ro.inner_bgr(frame.cpu().numpy(), layout))


def random_view(rs, layout, maps_cache):
    """A random frame of a random size in `layout` with random (cached) undistortion or random maps and a random window."""
    fh, fw = 2 * rs.randint(1, 30), 2 * rs.randint(1, 40)
    frame = torch.from_numpy(rc.frame(layout, int(rs.randint(1 << 30)), fh, fw)).cuda()
    kind = ("undistort", "random", "fisheye")[rs.randint(3)]
    mw, mh = rs.randint(1, 60), rs.randint(1, 50)
    key = (kind, mw, mh, fw, fh)
    if key not in maps_cache:
        mx, my = rc.float_maps(kind, mw, mh, fw, fh, int(rs.randint(1000)))
        maps_cache[key] = (eng.RemapMaps(mx, my), ro.convert_maps(mx, my))
    maps, fixed = maps_cache[key]
    w, h = rs.randint(1, mw + 1), rs.randint(1, mh + 1)
    x0, y0 = rs.randint(0, mw - w + 1), rs.randint(0, mh - h + 1)
    return eng.RemapView(frame, maps, x0, y0, w, h), fixed


def view_oracle(view, fixed, layout, W, H):
    img = ro.inner_bgr(view.frame.cpu().numpy(), layout)
    return ro.resize_planar(img, fixed[0], fixed[1], (view.x0, view.y0, view.w, view.h), W, H)


def plain_frames():
    """One plain frame of each of the 21 layouts."""
    pick = {c[1]: c for c in lc.CASES if c[0].endswith("_odd")}
    frames = {k: torch.from_numpy(np.ascontiguousarray(lc.case_input(c))).cuda() for k, c in pick.items()}
    for c in yc.CASES[:5]:
        frames.setdefault(c[1], torch.from_numpy(yc.case_input(c)).cuda())
    frames["bgr"] = torch.from_numpy(np.random.RandomState(5).randint(0, 256, (211, 157, 3)).astype(np.uint8)).cuda()
    for k in eng.BAYER_LAYOUTS:
        frames[k] = torch.from_numpy(np.random.RandomState(len(k)).randint(0, 256, (61, 83)).astype(np.uint8)).cuda()
    return frames


def plain_oracle(f, layout, W, H):
    if layout in eng.BAYER_LAYOUTS:
        return bo.resize_planar(f.cpu().numpy(), layout, W, H)
    import layout_oracle as lo
    return lo.resize_planar(f.cpu().numpy(), layout, W, H)


def test_mixed_batches_over_several_launches():
    """120 views of random layouts, sizes, maps and windows, runs of one kind long enough for several launches, with plain frames
    of all 21 layouts between them, in one call: each image equals the oracle, the remap alone too."""
    rs = np.random.RandomState(41)
    cache = {}
    layouts = ["bgr"] * 50 + [rc.LAYOUTS[rs.randint(21)] for _ in range(40)] + ["bayer_rg"] * 30
    views = [random_view(rs, lay, cache) for lay in layouts]
    plain = plain_frames()
    frames, lays, want = [], [], []
    for k, ((v, fixed), lay) in enumerate(zip(views, layouts)):
        frames.append(v)
        lays.append(lay)
        want.append(view_oracle(v, fixed, lay, 37, 29))
        if k >= 50 and k % 3 == 2:                      # after a 50-view BGR run: two launches of that kind
            p = rc.LAYOUTS[k % 21]
            frames.append(plain[p])
            lays.append(p)
            want.append(plain_oracle(plain[p], p, 37, 29))
    out = eng.resize_frames(frames, 37, 29, lays)
    for i, (w, lay) in enumerate(zip(want, lays)):
        assert np.array_equal(out[i].cpu().numpy(), w), (i, lay)
    rems = eng.remap_frames([v for v, _ in views], layouts)
    for (v, fixed), lay, r in zip(views, layouts, rems):
        img = ro.inner_bgr(v.frame.cpu().numpy(), lay)
        assert np.array_equal(r.cpu().numpy(), ro.remap_window(img, fixed[0], fixed[1], (v.x0, v.y0, v.w, v.h))), lay


def test_every_frame_and_map_form_gives_the_same_bytes(golden):
    for name in ("bgr_undistort", "nv12_convert_window", "gray_random", "bayer_rg_fisheye", "bgr_cv2fixed", "yuyv_undistort",
                 "bgr_junk"):
        c = [c for c in rc.CASES if c["name"] == name][0]
        W, H = c["target"]
        want = eng.resize_frames([case_view(c, golden)], W, H, c["layout"])
        frame = rc.case_frame(c)
        m1, m2 = rc.case_maps(c, golden)
        frame_forms = [frame, torch.from_numpy(frame).cuda()]
        if frame.ndim >= 2 and c["layout"] not in rc.YUV420:
            frame_forms.append(pitched(frame))
        d1 = torch.from_numpy(np.ascontiguousarray(m1)).cuda()
        d2 = None if m2 is None else torch.from_numpy(np.ascontiguousarray(m2.view(np.int16) if m2.dtype == np.uint16 else m2)).cuda()
        map_forms = [(m1, m2), (d1, d2)]
        if m2 is not None and m1.ndim == 2:                        # float planes as views into larger device tensors
            big = torch.zeros((2, m1.shape[0] + 2, m1.shape[1] + 5), dtype=torch.float32, device="cuda")
            big[0, 1:-1, 2:-3], big[1, 1:-1, 2:-3] = torch.from_numpy(m1), torch.from_numpy(m2)
            map_forms.append((big[0, 1:-1, 2:-3], big[1, 1:-1, 2:-3]))
        if m1.ndim == 3:                                           # [h, w, 2] as a non-contiguous (transposed) device tensor
            t = torch.from_numpy(np.ascontiguousarray(m1.transpose(1, 0, 2))).cuda().transpose(0, 1)
            map_forms.append((t, d2))
        if m2 is not None and m2.dtype == np.uint16:
            map_forms.append((m1, m2.view(np.int16)))
        for fi, f in enumerate(frame_forms):
            for mi, (a, b) in enumerate(map_forms):
                view = case_view(c, golden, f, eng.RemapMaps(a, b))
                assert torch.equal(eng.resize_frames([view], W, H, c["layout"]), want), (name, fi, mi)
        host_view = eng.RemapView(inner_frame(c, frame), eng.RemapMaps(m1, m2), *rc.view_window(c))
        assert torch.equal(eng.resize_frames([host_view], W, H, c["layout"]), want), name


@pytest.mark.parametrize("k", range(len(rc.ENCODE_CASES)))
def test_encode_jpeg_of_views_byte_identical_to_cv2(golden, k):
    name, q, s, region = rc.ENCODE_CASES[k]
    c = [c for c in rc.CASES if c["name"] == name][0]
    view = case_view(c, golden)
    regions = None if region is None else [(0,) + tuple(region)]
    got = eng.encode_jpeg([view], q, s, layout=c["layout"], regions=regions)[0]
    assert len(got) == int(golden["enc%d.len" % k])
    assert hashlib.sha256(got).digest() == golden["enc%d.sha" % k].tobytes()


def undistorted_modelzoo(golden_dir):
    """The bundled images with undistortion maps of their size (float form) and the oracle's corrected frames."""
    bgr = np.load(os.path.join(golden_dir, "frames_modelzoo.npz"))
    out = []
    for k, n in enumerate(lc.MODELZOO_FRAMES):
        img = bgr[n]
        h, w = img.shape[:2]
        kind = ("undistort", "fisheye")[k % 2]
        mx, my = rc.float_maps(kind, w, h, w, h, 0)
        fixed = ro.convert_maps(mx, my)
        out.append((n, img, eng.RemapMaps(mx, my), fixed, ro.remap(img, *fixed)))
    return out


def modelzoo_detector(golden_dir):
    import model.detector as det
    w = synth.load_modelzoo_weights(golden_dir)
    m = det.Detector(80, 3, True)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
    return m.cuda().eval()


def test_detect_frames_tiled_and_encode_on_views_equal_the_oracle_bgr(golden_dir):
    from utils import frames as uf
    m, cfg = modelzoo_detector(golden_dir), synth.coco_cfg()
    cases = undistorted_modelzoo(golden_dir)
    views, lays, bgrs = [], [], []
    for n, img, maps, fixed, corrected in cases:            # each image as BGR, and as a Bayer mosaic
        views.append(eng.RemapView(img, maps))
        lays.append("bgr")
        bgrs.append(corrected)
        raw = bo.mosaic(img, "bayer_bg")
        views.append(eng.RemapView(torch.from_numpy(raw).cuda(), maps))
        lays.append("bayer_bg")
        bgrs.append(ro.remap(bo.to_bgr(raw, "bayer_bg"), *fixed))
    got = uf.detect_frames(m, views, cfg, conf_thres=0.3, iou_thres=0.4, layout=lays)
    want = uf.detect_frames(m, bgrs, cfg, conf_thres=0.3, iou_thres=0.4, layout="bgr")
    for a, b in zip(got, want):
        assert a.dtype == torch.float64 and torch.equal(a, b)
    assert sum(g.shape[0] for g in got) > 0
    tiled = uf.detect_tiled(m, views, cfg, 3, 2, 0.2, True, layout=lays, conf_thres=0.2)
    tiled_bgr = uf.detect_tiled(m, bgrs, cfg, 3, 2, 0.2, True, layout="bgr", conf_thres=0.2)
    for a, b in zip(tiled, tiled_bgr):
        assert a.dtype == torch.float64 and torch.equal(a, b)
    assert sum(a.shape[0] for a in tiled) > 0
    win = eng.crop_frame(views[0], "bgr", 31, 17, 301, 251)
    regs = uf.detect_regions(m, [win], cfg, [[(0, 0, 301, 251), (7, 9, 151, 121)]], layout="bgr", conf_thres=0.2)
    regs_bgr = uf.detect_regions(m, [np.ascontiguousarray(bgrs[0][17:268, 31:332])], cfg, [[(0, 0, 301, 251), (7, 9, 151, 121)]],
                                 layout="bgr", conf_thres=0.2)
    assert torch.equal(regs[0], regs_bgr[0])
    files = uf.encode_detections([views[0], win, views[1]], [got[0], regs[0], got[1]], layout=["bgr", "bgr", "bayer_bg"],
                                 quality=90)
    files_bgr = uf.encode_detections([bgrs[0], np.ascontiguousarray(bgrs[0][17:268, 31:332]), bgrs[1]],
                                     [got[0], regs[0], got[1]], quality=90)
    assert files == files_bgr and len(files[0]) == got[0].shape[0]
    whole = eng.encode_jpeg(views + bgrs, 95, "420", layout=lays + ["bgr"] * len(bgrs))
    assert whole[:len(views)] == whole[len(views):]


def test_track_frames_on_views_equal_the_oracle_bgr(golden_dir):
    """A zoom and pan over undistorted views of the two bundled images in two streams, against the same calls on the oracle's
    corrected windows, step by step."""
    from utils.tracking import track_frames
    m, cfg = modelzoo_detector(golden_dir), synth.coco_cfg()
    cases = undistorted_modelzoo(golden_dir)
    tracker, tracker_bgr = eng.Tracker("cuda", 2, 64), eng.Tracker("cuda", 2, 64)
    total = 0
    for k in range(6):
        frames, frames_bgr = [], []
        for n, img, maps, _, corrected in cases:
            h, w = img.shape[:2]
            x0, y0 = 3 * k, 5 * k
            frames.append(eng.crop_frame(eng.RemapView(torch.from_numpy(img).cuda(), maps), "bgr", x0, y0, w - 2 * x0, h - y0 - k))
            frames_bgr.append(np.ascontiguousarray(corrected[y0:h - k, x0:w - x0]))
        got = track_frames(m, tracker, frames, cfg, layout="bgr")
        want = track_frames(m, tracker_bgr, frames_bgr, cfg, layout="bgr")
        for a, b in zip(got, want):
            assert a.dtype == torch.float64 and torch.equal(a, b), k
        total += sum(a.shape[0] for a in got)
    assert total > 0

"""Warped views on the device (resize_frames through yfv2_resize_warp_u8, warp_frames through yfv2_warp_u8) against the frozen
cv2.cvtColor + cv2.warpAffine / cv2.warpPerspective + crop + cv2.resize / cv2.imencode outputs and the numpy oracle, bit for bit:
every case in every inner kind, batches mixing differently warped views with plain frames of every layout over several launches,
the same warp through RemapView and the oracle's fixed maps, and detect_frames, detect_tiled, detect_regions, track_frames,
encode_jpeg and encode_detections on warped views of the bundled images."""
import hashlib
import os

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import bayer_oracle as bo
import layout_cases as lc
import remap_oracle as ro
import synth
import warp_cases as wc
import warp_oracle as wo
import yfv2_engine as eng
import yuv_cases as yc
from oracle import resize as ore

pytestmark = pytest.mark.gpu


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def hwc(planar):
    return planar.permute(1, 2, 0).contiguous().cpu().numpy()


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "warp_cases.npz"))


def case_view(c, golden, frame=None):
    frame = torch.from_numpy(wc.case_frame(c)).cuda() if frame is None else frame
    inner = frame if c["inner"] is None else eng.crop_frame(frame, c["layout"], *c["inner"])
    return eng.WarpView(inner, wc.case_matrix(c, golden), c["dsize"], *wc.view_window(c), inverse=c["inverse"])


@pytest.mark.parametrize("c", wc.CASES, ids=[c["name"] for c in wc.CASES])
def test_bit_exact_against_cv2_golden_and_oracle(golden, c):
    name, (W, H) = c["name"], c["target"]
    view = case_view(c, golden)
    out = eng.resize_frames([view], W, H, c["layout"])
    assert out.shape == (1, 3, H, W) and out.dtype == torch.uint8
    got = hwc(out[0])
    if name + "_out" in golden:
        assert np.array_equal(got, golden[name + "_out"])
    assert np.array_equal(sha(got), golden[name + "_sha256"])
    img = ro.inner_bgr(wc.case_frame(c), c["layout"], c["inner"])
    M = wc.case_matrix(c, golden)
    assert np.array_equal(out[0].cpu().numpy(), wo.resize_planar(img, M, c["dsize"], wc.view_window(c), W, H, c["inverse"]))
    warp = eng.warp_frames([view], c["layout"])[0]
    assert warp.shape == (view.h, view.w, 3) and warp.dtype == torch.uint8 and warp.is_cuda
    warp = warp.cpu().numpy()
    if name + "_warp" in golden:
        assert np.array_equal(warp, golden[name + "_warp"])
    assert np.array_equal(sha(warp), golden[name + "_warp_sha256"])


def test_host_frames_and_lists_give_the_same_bytes(golden):
    """A host frame and a nested-list matrix give the bytes of a device frame and a numpy matrix."""
    for name in ("bgr_rot_any", "nv12_inner_crop", "bayer_bg_inner_window_persp", "gray_scale_up"):
        c = [c for c in wc.CASES if c["name"] == name][0]
        W, H = c["target"]
        want = eng.resize_frames([case_view(c, golden)], W, H, c["layout"])
        frame = wc.case_frame(c)
        inner = frame if c["inner"] is None else eng.crop_frame(frame, c["layout"], *c["inner"])
        v = eng.WarpView(inner, wc.case_matrix(c, golden).tolist(), c["dsize"], *wc.view_window(c), inverse=c["inverse"])
        assert torch.equal(eng.resize_frames([v], W, H, c["layout"]), want), name


def random_view(rs, layout):
    """A random frame of a random size in `layout` with a random affine or perspective matrix, output size and window."""
    fh, fw = 2 * rs.randint(1, 30), 2 * rs.randint(1, 40)
    frame = torch.from_numpy(wc.frame(layout, int(rs.randint(1 << 30)), fh, fw)).cuda()
    dw, dh = rs.randint(1, 70), rs.randint(1, 60)
    if rs.randint(2):
        M = wc.rotation(rs.uniform(0, fw), rs.uniform(0, fh), rs.uniform(-180, 180), rs.uniform(0.3, 2.5))
        M[0, 1] += rs.uniform(-0.2, 0.2)
    else:
        M = wc.quad_homography(fw, fh, rs.uniform(-0.3, 0.3, (4, 2)))
    w, h = rs.randint(1, dw + 1), rs.randint(1, dh + 1)
    x0, y0 = rs.randint(0, dw - w + 1), rs.randint(0, dh - h + 1)
    return eng.WarpView(frame, M, (dw, dh), x0, y0, w, h, inverse=bool(rs.randint(2)))


def view_bgr(view, layout):
    img = ro.inner_bgr(view.frame.cpu().numpy(), layout)
    M = np.array(view.m).reshape(3 if view.perspective else 2, 3)
    return wo.warp_window(img, M, (view.dw, view.dh), (view.x0, view.y0, view.w, view.h), view.inverse)


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


def test_mixed_batches_with_a_matrix_per_frame_over_several_launches():
    """130 views, each with its own matrix, output size and window: a 70-view BGR run and a 40-view Bayer run (each more than one
    launch chunk), random layouts between, with plain frames of all 21 layouts among them, in one call; the warp alone too."""
    rs = np.random.RandomState(43)
    layouts = ["bgr"] * 70 + [wc.LAYOUTS[rs.randint(21)] for _ in range(20)] + ["bayer_rg"] * 40
    views = [random_view(rs, lay) for lay in layouts]
    plain = plain_frames()
    frames, lays, want = [], [], []
    for k, (v, lay) in enumerate(zip(views, layouts)):
        frames.append(v)
        lays.append(lay)
        want.append(ore.resize_bgr_planar(view_bgr(v, lay), 37, 29))
        if 70 <= k < 90 and k % 3 == 2:
            p = wc.LAYOUTS[k % 21]
            frames.append(plain[p])
            lays.append(p)
            want.append(plain_oracle(plain[p], p, 37, 29))
    out = eng.resize_frames(frames, 37, 29, lays)
    for i, (w, lay) in enumerate(zip(want, lays)):
        assert np.array_equal(out[i].cpu().numpy(), w), (i, lay)
    warps = eng.warp_frames(views, layouts)
    for v, lay, r in zip(views, layouts, warps):
        assert np.array_equal(r.cpu().numpy(), view_bgr(v, lay)), lay


@pytest.mark.parametrize("name", ["bgr_rot", "nv12_persp_window", "bgr_birdseye", "bayer_gr_ea_inner_window",
                                  "bgr_horizon_row", "yuyv_shear_inverse", "bgr_affine_ties", "gray_persp_ties"])
def test_warp_view_equals_remap_view_through_the_oracles_maps(golden, name):
    """The same warp through the old path (RemapView over the oracle's fixed maps of the warp) and the new one: identical bytes."""
    c = [c for c in wc.CASES if c["name"] == name][0]
    W, H = c["target"]
    view = case_view(c, golden)
    persp, m = wo.dst_to_src(wc.case_matrix(c, golden), c["inverse"])
    xy, code = wo.warp_maps(m, persp, 0, 0, *c["dsize"])
    rview = eng.RemapView(view.frame, eng.RemapMaps(xy, code), *wc.view_window(c))
    assert torch.equal(eng.resize_frames([view], W, H, c["layout"]), eng.resize_frames([rview], W, H, c["layout"]))
    assert torch.equal(eng.warp_frames([view], c["layout"])[0], eng.remap_frames([rview], c["layout"])[0])


@pytest.mark.parametrize("k", range(len(wc.ENCODE_CASES)))
def test_encode_jpeg_of_views_byte_identical_to_cv2(golden, k):
    name, q, s, region = wc.ENCODE_CASES[k]
    c = [c for c in wc.CASES if c["name"] == name][0]
    view = case_view(c, golden)
    regions = None if region is None else [(0,) + tuple(region)]
    got = eng.encode_jpeg([view], q, s, layout=c["layout"], regions=regions)[0]
    assert len(got) == int(golden["enc%d.len" % k])
    assert hashlib.sha256(got).digest() == golden["enc%d.sha" % k].tobytes()


def warped_modelzoo(golden_dir):
    """The bundled images with a rotation (affine) or a de-skew (perspective) of their size, and the oracle's warped frames."""
    bgr = np.load(os.path.join(golden_dir, "frames_modelzoo.npz"))
    out = []
    for k, n in enumerate(lc.MODELZOO_FRAMES):
        img = bgr[n]
        h, w = img.shape[:2]
        M = (wc.rotation(w / 2, h / 2, 8.0, 0.95) if k % 2 == 0 else
             wc.quad_homography(w, h, [[0.04, 0.02], [-0.03, 0.0], [0.0, 0.0], [0.02, -0.03]]))
        out.append((n, img, M, (w, h), wo.warp_window(img, M, (w, h))))
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
    views, lays, bgrs = [], [], []
    for n, img, M, dsize, warped in warped_modelzoo(golden_dir):      # each image as BGR, and as a Bayer mosaic
        views.append(eng.WarpView(img, M, dsize))
        lays.append("bgr")
        bgrs.append(warped)
        raw = bo.mosaic(img, "bayer_bg")
        views.append(eng.WarpView(torch.from_numpy(raw).cuda(), M, dsize))
        lays.append("bayer_bg")
        bgrs.append(wo.warp_window(bo.to_bgr(raw, "bayer_bg"), M, dsize))
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


def test_track_frames_on_views_with_a_matrix_per_frame_equal_the_oracle_bgr(golden_dir):
    """Digital stabilisation: two streams whose matrix changes on every frame (a small rotation and shift), cropped by a zoom,
    against the same calls on the oracle's warped windows, step by step."""
    from utils.tracking import track_frames
    m, cfg = modelzoo_detector(golden_dir), synth.coco_cfg()
    cases = warped_modelzoo(golden_dir)
    tracker, tracker_bgr = eng.Tracker("cuda", 2, 64), eng.Tracker("cuda", 2, 64)
    total = 0
    for k in range(6):
        frames, frames_bgr = [], []
        for n, img, _, _, _ in cases:
            h, w = img.shape[:2]
            M = wc.rotation(w / 2 + k, h / 2 - k, 1.5 * k - 4, 1.0)
            x0, y0 = 3 * k, 5 * k
            frames.append(eng.crop_frame(eng.WarpView(torch.from_numpy(img).cuda(), M, (w, h)), "bgr", x0, y0, w - 2 * x0,
                                         h - y0 - k))
            frames_bgr.append(np.ascontiguousarray(wo.warp_window(img, M, (w, h))[y0:h - k, x0:w - x0]))
        got = track_frames(m, tracker, frames, cfg, layout="bgr")
        want = track_frames(m, tracker_bgr, frames_bgr, cfg, layout="bgr")
        for a, b in zip(got, want):
            assert a.dtype == torch.float64 and torch.equal(a, b), k
        total += sum(a.shape[0] for a in got)
    assert total > 0

"""Detection on regions of frames on the device: yfv2_merge_regions against tests/region_oracle.py bit for bit (rows, counts and
source indices, both metrics), crop_frame + resize_frames against the numpy crop's oracle bytes in all 13 layouts, detect_regions
with one whole-frame region equal to detect_frames, and detect_tiled equal to the oracle applied to the per-region detections."""
import os

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import layout_cases as lc
import layout_oracle as lo
import region_cases as rc
import region_oracle as ro
import synth
import yfv2_engine as eng
import yuv_cases as yc

pytestmark = pytest.mark.gpu


def kernel(dets, counts, regions, F, W, H, thr, metric, max_det):
    out, n, src = eng.merge_regions(torch.from_numpy(np.ascontiguousarray(dets)).cuda(), torch.from_numpy(counts).cuda(), regions, F,
                                    W, H, thr, metric, max_det)
    return out.cpu().numpy(), n.cpu().numpy(), src.cpu().numpy()


def same(got, want):
    """Bit for bit: float64 rows compared as bytes (so NaN, -0 and +0 count), counts and kept_src as integers."""
    (o, n, s), (wo, wn, ws) = got, want
    assert np.array_equal(n, wn), (n, wn)
    assert np.array_equal(s, ws)
    assert np.array_equal(o.view(np.uint64), wo.view(np.uint64))


@pytest.mark.parametrize("case", rc.hand_cases(), ids=[c[0] for c in rc.hand_cases()])
def test_hand_cases_bit_exact(case):
    args = case[1:]
    same(kernel(*args), ro.merge(*args))


@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("max_det", [1, 300, 4096])
def test_random_frames_bit_exact(metric, max_det):
    """300 frames with 0-27 regions each, 0-40 rows per region, coarse boxes and quantised conf (many overlaps and ties)."""
    d, n, r = rc.random_case(11 + metric)
    for thr in (0.3, 0.7):
        same(kernel(d, n, r, 300, 352, 352, thr, metric, max_det), ro.merge(d, n, r, 300, 352, 352, thr, metric, max_det))


@pytest.mark.parametrize("metric", [0, 1])
def test_dense_frames_of_27_regions_of_300_rows(metric):
    """8100 candidates per frame, the sort's largest size, and counts that hold the garbage rows past max_det_in out of reach."""
    d, n, r = rc.random_case(21, F=3, max_regions=27, max_det_in=300, dense=True)
    for max_det in (1000, 4096):
        same(kernel(d, n, r, 3, 352, 352, 0.5, metric, max_det), ro.merge(d, n, r, 3, 352, 352, 0.5, metric, max_det))


def test_the_candidate_limit():
    """32 regions of 256 rows (8192 candidates) are allowed and exact; a 33rd region is refused before anything runs."""
    d, n, r = rc.random_case(23, F=2, max_regions=32, max_det_in=256, dense=True)
    same(kernel(d, n, r, 2, 352, 352, 0.5, 1, 4096), ro.merge(d, n, r, 2, 352, 352, 0.5, 1, 4096))
    d = np.concatenate([d[:33], d[32:]])
    n = np.concatenate([n[:33], n[32:]])
    r = [(0,) + x[1:] for x in r[:33]] + r[32:]
    with pytest.raises(eng.Yfv2Error, match="8192"):
        kernel(d, n, r, 2, 352, 352, 0.5, 1, 4096)


def test_many_frames_span_several_launches():
    """1000 frames (eight launches of 128), sizes of region lists from 0 to 8, counts past max_det_in and negative ones clamped."""
    d, n, r = rc.random_case(29, F=1000, max_regions=8, max_det_in=40, max_rows=40)
    n = n.copy()
    n[::7] = 1000
    n[3::11] = -5
    same(kernel(d, n, r, 1000, 352, 352, 0.5, 1, 64), ro.merge(d, n, r, 1000, 352, 352, 0.5, 1, 64))


# ---- crops ---------------------------------------------------------------------------------------------------------------------------
def crop_sources():
    """One frame of every layout: 4:2:0 from tests/yuv_cases.py, the others from tests/layout_cases.py (odd sizes where allowed)."""
    out = {}
    for c in yc.CASES:
        if c[5] is None and c[1] not in out and c[3][0] >= 300:
            out[c[1]] = yc.case_input(c)
    for c in lc.CASES:
        if c[0] == c[1] + "_odd":
            out[c[1]] = lc.case_input(c)
    out["bgr"] = np.random.RandomState(31).randint(0, 256, (177, 333, 3)).astype(np.uint8)
    assert sorted(out) == sorted(eng.LAYOUTS)
    return out


@pytest.mark.parametrize("layout", eng.LAYOUTS)
def test_crop_then_resize_equals_the_oracle_of_the_numpy_crop(layout):
    from oracle import resize as ore
    frame = crop_sources()[layout]
    fh, fw = eng.frame_size(frame, layout)
    dev = torch.from_numpy(np.ascontiguousarray(frame)).cuda()
    windows = [(0, 0, fw, fh), (0, 0, 2, 2), (fw - 2, fh - 2, 2, 2), (2, 4, 40, 32), (fw - 100, fh - 60, 100, 60), (12, 30, fw - 30, 48)]
    if layout not in eng.YUV420_LAYOUTS:
        windows += [(1 if layout not in eng.YUV422_LAYOUTS else 2, 3, 66, 17), (fw - 37 + (layout in eng.YUV422_LAYOUTS), 5, 36, 1)]
    bgr = lo.to_bgr(frame, layout)
    for (x0, y0, w, h) in windows:
        want = {(W, H): ore.resize_bgr_planar(np.ascontiguousarray(bgr[y0:y0 + h, x0:x0 + w]), W, H) for W, H in ((352, 352), (37, 29))}
        for src in (frame, dev):
            crop = eng.crop_frame(src, layout, x0, y0, w, h)
            for W, H in ((352, 352), (37, 29)):
                got = eng.resize_frames([crop], W, H, layout)[0].cpu().numpy()
                assert np.array_equal(got, want[W, H]), (layout, x0, y0, w, h, W, H)


# ---- detect_regions / detect_tiled ---------------------------------------------------------------------------------------------------
def modelzoo_detector(golden_dir):
    import model.detector as det
    w = synth.load_modelzoo_weights(golden_dir)
    m = det.Detector(80, 3, True)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
    return m.cuda().eval()


@pytest.fixture(scope="module")
def zoo(golden_dir):
    golden = np.load(os.path.join(golden_dir, "layout_cases.npz"))
    bgr = np.load(os.path.join(golden_dir, "frames_modelzoo.npz"))
    yuv = np.load(os.path.join(golden_dir, "yuv_cases.npz"))
    return modelzoo_detector(golden_dir), synth.coco_cfg(), golden, bgr, yuv


def bundled_frames(zoo, layout):
    _, _, golden, bgr, yuv = zoo
    if layout == "bgr":
        return [bgr[n] for n in lc.MODELZOO_FRAMES]
    if layout in eng.YUV420_LAYOUTS:
        frames = []
        for n in lc.MODELZOO_FRAMES:
            i420 = yuv[n + "_i420"]
            h, w = i420.shape[0] // 3 * 2, i420.shape[1]
            if layout == "i420":
                frames.append(i420)
            elif layout == "nv12":
                frames.append(yc.i420_to_nv12(i420))
            else:
                q = (h // 2) * (w // 2)
                flat = i420.reshape(-1)
                u, v = flat[h * w:h * w + q].reshape(h // 2, w // 2), flat[h * w + q:].reshape(h // 2, w // 2)
                frames.append(yc.single_buffer((i420[:h], u, v), layout) if layout == "yv12"
                              else np.concatenate([i420[:h], np.stack([v, u], -1).reshape(h // 2, w)]))
        return frames
    return [lc.bundled(golden, bgr, n, layout) for n in lc.MODELZOO_FRAMES]


@pytest.mark.parametrize("layout", eng.LAYOUTS)
def test_one_whole_frame_region_is_detect_frames(zoo, layout):
    from utils import frames as uf
    m, cfg = zoo[0], zoo[1]
    frames = bundled_frames(zoo, layout)
    want = uf.detect_frames(m, frames, cfg, conf_thres=0.3, iou_thres=0.4, layout=layout)
    regions = [[(0, 0) + tuple(eng.frame_size(f, layout))[::-1]] for f in frames]
    got = uf.detect_regions(m, frames, cfg, regions, conf_thres=0.3, iou_thres=0.4, layout=layout)
    assert len(got) == len(want)
    for a, b in zip(got, want):
        assert a.dtype == torch.float64 and torch.equal(a, b)
    assert sum(a.shape[0] for a in got) > 0


@pytest.mark.parametrize("layout,merge", [("bgr", "ios"), ("bgr", "iou"), ("nv12", "ios"), ("yuyv", "ios"), ("rgb_chw", "iou")])
def test_detect_tiled_is_the_oracle_of_the_per_region_detections(zoo, layout, merge):
    from utils import frames as uf
    m, cfg = zoo[0], zoo[1]
    frames = bundled_frames(zoo, layout)
    regions = [uf.tile_regions(*eng.frame_size(f, layout)[::-1], 3, 2, 0.2, True, layout) for f in frames]
    got = uf.detect_tiled(m, frames, cfg, 3, 2, 0.2, True, layout=layout, merge=merge, merge_thres=0.5, conf_thres=0.2)
    again = uf.detect_tiled(m, frames, cfg, 3, 2, 0.2, True, layout=layout, merge=merge, merge_thres=0.5, conf_thres=0.2, batch=7)
    assert all(torch.equal(a, b) for a, b in zip(got, again))
    crops, descs = [], []
    for i, (f, regs) in enumerate(zip(frames, regions)):
        for reg in regs:
            crops.append(eng.crop_frame(f, layout, *reg))
            descs.append((i,) + tuple(reg))
    x = eng.resize_frames(crops, 352, 352, layout)
    with torch.no_grad():
        out, n, _ = eng.decode_nms(m(x), cfg, 0.2, 0.4)
    want, wn, _ = ro.merge(out.cpu().numpy(), n.cpu().numpy(), descs, len(frames), 352, 352, 0.5, merge, 1000)
    for i, g in enumerate(got):
        assert g.dtype == torch.float64 and g.shape[0] == wn[i]
        assert np.array_equal(g.numpy().view(np.uint64), want[i, :wn[i]].view(np.uint64))
    assert sum(g.shape[0] for g in got) > 0
    print("detect_tiled(%s, %s): %s" % (layout, merge, [g.shape[0] for g in got]))

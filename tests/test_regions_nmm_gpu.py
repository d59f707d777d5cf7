"""Greedy non-maximum merging of the cross-region merge on the device: yfv2_merge_regions_nmm against
tests/region_nmm_oracle.py bit for bit (float64 rows as bytes, counts, kept_src and merged), and on every case the invariants against
yfv2_merge_regions (counts, conf, cls and kept_src equal; each box contains the NMS box), then detect_tiled(merge_mode="nmm") on
the bundled images against the oracle over the per-region detections."""
import os

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import region_cases as rc
import region_nmm_cases as nc
import region_nmm_oracle as rno
import synth
import yfv2_engine as eng

pytestmark = pytest.mark.gpu


def kernels(dets, counts, regions, F, W, H, thr, metric, max_det):
    """(NMM out, counts, kept_src, merged) and the NMS merge's (out, counts, kept_src) of the same device input."""
    d, n = torch.from_numpy(np.ascontiguousarray(dets)).cuda(), torch.from_numpy(np.ascontiguousarray(counts)).cuda()
    nmm = eng.merge_regions(d, n, regions, F, W, H, thr, metric, max_det, mode="nmm", want_merged=True)
    nms = eng.merge_regions(d, n, regions, F, W, H, thr, metric, max_det)
    return [t.cpu().numpy() for t in nmm], [t.cpu().numpy() for t in nms]


def check(dets, counts, regions, F, W, H, thr, metric, max_det):
    (o, n, s, m), (wo, wn, ws) = kernels(dets, counts, regions, F, W, H, thr, metric, max_det)
    # against yfv2_merge_regions: the same rows, only the boxes grown
    assert np.array_equal(n, wn) and np.array_equal(s, ws)
    assert np.array_equal(o[..., 4:].view(np.uint64), wo[..., 4:].view(np.uint64))
    with np.errstate(invalid="ignore"):
        inside = (o[..., :2] <= wo[..., :2]).all(-1) & (o[..., 2:4] >= wo[..., 2:4]).all(-1)
    assert (inside | np.isnan(o[..., :4]).any(-1) | np.isnan(wo[..., :4]).any(-1)).all()
    # against the oracle, bit for bit
    eo, en, es, em = rno.merge_nmm(dets, counts, regions, F, W, H, thr, metric, max_det)
    assert np.array_equal(n, en) and np.array_equal(s, es)
    assert np.array_equal(m, em)
    assert np.array_equal(o.view(np.uint64), eo.view(np.uint64))
    return m


@pytest.mark.parametrize("case", nc.all_hand_cases(), ids=[c[0] for c in nc.all_hand_cases()])
def test_hand_cases_bit_exact(case):
    check(*case[1:])


def test_merged_is_optional():
    _, d, n, r, F, W, H, thr, metric, max_det = nc.hand_cases()[0]
    dd, nn = torch.from_numpy(d).cuda(), torch.from_numpy(n).cuda()
    a = eng.merge_regions(dd, nn, r, F, W, H, thr, metric, max_det, mode="nmm")
    b = eng.merge_regions(dd, nn, r, F, W, H, thr, metric, max_det, mode="nmm", want_merged=True)
    assert len(a) == 3 and len(b) == 4 and all(torch.equal(x, y) for x, y in zip(a, b[:3]))


@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("max_det", [1, 300, 4096])
def test_random_frames_bit_exact(metric, max_det):
    """300 frames with 0-27 regions each, 0-40 rows per region, coarse boxes and quantised conf (many overlaps and ties)."""
    d, n, r = rc.random_case(11 + metric)
    for thr in (0.3, 0.7):
        m = check(d, n, r, 300, 352, 352, thr, metric, max_det)
        if max_det > 1:
            assert m.any()


@pytest.mark.parametrize("metric", [0, 1])
def test_dense_frames_of_27_regions_of_300_rows(metric):
    """8100 candidates per frame; at max_det 1000 most rows come after the cap, and rows after it are absorbed."""
    d, n, r = rc.random_case(21, F=3, max_regions=27, max_det_in=300, dense=True)
    for max_det in (1, 1000, 4096):
        m = check(d, n, r, 3, 352, 352, 0.5, metric, max_det)
        if max_det == 1:
            assert m[:, 0].any()


def test_the_candidate_limit():
    """32 regions of 256 rows (8192 candidates) at max_det 4096 and 1: the largest shared-memory layout, and one absorber for all."""
    d, n, r = rc.random_case(23, F=2, max_regions=32, max_det_in=256, dense=True)
    for max_det in (4096, 1):
        check(d, n, r, 2, 352, 352, 0.5, 1, max_det)
    # every row one class and one box grown from the first: 8191 rows absorbed by a single output row, folded in order
    d2 = d.copy()
    d2[..., 5] = 0.0
    check(d2, n, r, 2, 352, 352, -1.0, 0, 1)


def test_many_frames_span_several_launches():
    """1000 frames (eight launches of 128), sizes of region lists from 0 to 8, counts past max_det_in and negative ones clamped."""
    d, n, r = rc.random_case(29, F=1000, max_regions=8, max_det_in=40, max_rows=40)
    n = n.copy()
    n[::7] = 1000
    n[3::11] = -5
    check(d, n, r, 1000, 352, 352, 0.5, 1, 64)


# ---- detect_tiled(merge_mode="nmm") -------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def zoo(golden_dir):
    import model.detector as det
    w = synth.load_modelzoo_weights(golden_dir)
    m = det.Detector(80, 3, True)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
    bgr = np.load(os.path.join(golden_dir, "frames_modelzoo.npz"))
    return m.cuda().eval(), synth.coco_cfg(), bgr


@pytest.mark.parametrize("merge", ["ios", "iou"])
def test_detect_tiled_nmm_is_the_oracle_of_the_per_region_detections(zoo, merge):
    import layout_cases as lc
    from utils import frames as uf
    m, cfg, bgr = zoo
    frames = [bgr[k] for k in lc.MODELZOO_FRAMES]
    regions = [uf.tile_regions(f.shape[1], f.shape[0], 3, 2, 0.2, True) for f in frames]
    got = uf.detect_tiled(m, frames, cfg, 3, 2, 0.2, True, merge=merge, merge_thres=0.5, conf_thres=0.2, merge_mode="nmm")
    again = uf.detect_tiled(m, frames, cfg, 3, 2, 0.2, True, merge=merge, merge_thres=0.5, conf_thres=0.2, merge_mode="nmm",
                            batch=7)
    assert all(torch.equal(a, b) for a, b in zip(got, again))
    crops, descs = [], []
    for i, (f, regs) in enumerate(zip(frames, regions)):
        for reg in regs:
            crops.append(eng.crop_frame(f, "bgr", *reg))
            descs.append((i,) + tuple(reg))
    x = eng.resize_frames(crops, 352, 352, "bgr")
    with torch.no_grad():
        out, n, _ = eng.decode_nms(m(x), cfg, 0.2, 0.4)
    want, wn, _, wm = rno.merge_nmm(out.cpu().numpy(), n.cpu().numpy(), descs, len(frames), 352, 352, 0.5, merge, 1000)
    nms = uf.detect_tiled(m, frames, cfg, 3, 2, 0.2, True, merge=merge, merge_thres=0.5, conf_thres=0.2)
    for i, g in enumerate(got):
        assert g.dtype == torch.float64 and g.shape[0] == wn[i]
        assert np.array_equal(g.numpy().view(np.uint64), want[i, :wn[i]].view(np.uint64))
        assert torch.equal(g[:, 4:], nms[i][:, 4:])
    assert sum(g.shape[0] for g in got) > 0
    print("detect_tiled(nmm, %s): rows %s, rows merged %d" % (merge, [g.shape[0] for g in got], int(wm.sum())))

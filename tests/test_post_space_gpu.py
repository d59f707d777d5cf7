"""Device NMS and fused decode + NMS across the code paths k_post.cu picks from its arguments: caps (max_det 1 .. the largest that
fits in shared memory), both suppression policies (dense scan / per-class kept lists), every sort size, the exact IoU fallback,
thresholds outside (0, 1), degenerate boxes, score ties at chunk and cap boundaries, every candidate-generation path of the
fused kernel, and the runtime switches of INTEGRATION.md §5.  Every case is bit-exact against oracle.post (rows and kept
indices) on the same input tensor; fused cases are also bit-identical to yfv2_decode followed by yfv2_nms.
tests/post_space.py restates the host-side choices, and the tests assert that each input lands on the side it was built for."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import post_space as ps
import synth
import yfv2_engine as eng
from oracle import post as opost

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def check_nms(d, ct, it, max_det=300, max_wh=4096.0):
    """yfv2_nms on d [N, M, 5+C] (numpy) against the oracle, bit for bit.  Returns the counts."""
    out, counts, idx = eng.nms(torch.from_numpy(d).cuda(), ct, it, max_det=max_det, max_wh=max_wh)
    rows, oidx = opost.nms(torch.from_numpy(d), ct, it, return_indices=True, max_det=max_det, max_wh=max_wh)
    out, counts, idx = out.cpu().numpy(), counts.cpu().numpy(), idx.cpu().numpy()
    for i in range(d.shape[0]):
        c = int(counts[i])
        tag = (ct, it, max_det, max_wh, i)
        assert c == rows[i].shape[0], tag
        assert np.array_equal(out[i, :c], rows[i].numpy()), tag
        assert np.array_equal(idx[i, :c], oidx[i]), tag
        assert np.all(out[i, c:] == 0) and np.all(idx[i, c:] == -1), tag
    return counts


def check_fused(preds, cfg, ct, it, max_det=300, max_wh=4096.0):
    """yfv2_decode_nms == yfv2_decode -> yfv2_nms bit for bit, and that NMS bit-exact against the oracle on the decoded tensor.
    Returns (decoded tensor on the host, counts)."""
    d = eng.decode(preds, cfg)
    out, counts, idx = eng.nms(d, ct, it, max_det=max_det, max_wh=max_wh)
    f_out, f_counts, f_idx = eng.decode_nms(preds, cfg, ct, it, max_det=max_det, want_idx=True, max_wh=max_wh)
    tag = (preds[1].shape[1], preds[2].shape[1], ct, it, max_det, max_wh)
    assert torch.equal(counts, f_counts), tag
    assert torch.equal(idx, f_idx), tag
    assert torch.equal(out, f_out), tag
    dh = d.cpu().numpy()
    check_nms(dh, ct, it, max_det, max_wh)
    return dh, counts.cpu().numpy()


def cfg_for(A, C, H, W):
    cfg = synth.coco_cfg(W, H, C)
    cfg["anchor_num"] = A
    rs = np.random.RandomState(A * 1000 + C)
    cfg["anchors"] = [float(v) for v in np.round(rs.uniform(8, 300, 4 * A), 2)]
    return cfg


def heads(seed, n, H, W, A, C):
    return [p.numpy().copy() for p in synth.make_head_logits(seed, n, H, W, classes=C, anchor_num=A)]


def to_dev(hs):
    return [torch.from_numpy(h).cuda() for h in hs]


# ---------------------------------------------------------------------------------------------------------------------------
# caps x suppression policy

def policy_inputs():
    """name -> one image [1, M, 85] and a predicate (max_det, max_wh) -> whether the per-class lists are meant to be taken."""
    big = lambda md: md >= ps.LIST_MIN_DET                                                   # noqa: E731
    wide = ps.random_dets(105, 1, 6000, side=640.0)
    wide[0, ::3, 2:4] += 60000.0                              # boxes far wider than the class offset: neighbouring classes overlap
    wide[0, :, 0] *= 3.0
    return {
        "m6000_640": (ps.random_dets(101, 1, 6000, side=640.0), lambda md, wh: big(md) and wh == 4096.0),   # outside +-512
        "m6000_352": (ps.random_dets(102, 1, 6000, side=352.0, size=100.0), lambda md, wh: big(md) and wh > 0),
        "m6000_majority": (ps.random_dets(103, 1, 6000, side=640.0, majority=3), lambda md, wh: False),
        "m6000_half": (ps.random_dets(104, 1, 6000, side=640.0, half=True), lambda md, wh: big(md) and wh == 4096.0),
        "m6000_wide": (wide, lambda md, wh: False),
        "m1815": (ps.random_dets(106, 1, 1815, side=352.0), lambda md, wh: False),           # no room for the lists
        "m2048": (ps.random_dets(107, 1, 2048, side=352.0), lambda md, wh: False),           # no padding at all
    }


CAPS = [1, 63, 64, 65, 300, 513, 1000, 4096]


def run_caps_and_policy(lists_always=False, names=None, caps=None, max_whs=(4096.0, 1024.0, 0.0), it=0.45):
    """Every (input, cap, max_wh) bit-exact against the oracle; caps that do not fit in shared memory are replaced by the largest
    that does.  Returns the number of cases on the per-class list path."""
    n_lists = 0
    for name, (d, meant) in policy_inputs().items():
        if names is not None and name not in names:
            continue
        M = d.shape[1]
        for md in sorted(set(min(c, ps.largest_cap(M)) for c in (caps or CAPS + [ps.largest_cap(M)]))):
            for wh in max_whs:
                lists = ps.by_class(d[0], 0.001, it, md, wh, lists_always)
                if not lists_always:
                    assert lists == meant(md, wh), (name, md, wh)                  # the input is on the side it was built for
                n_lists += lists
                counts = check_nms(d, 0.001, it, md, wh)
                assert int(counts[0]) > 0
    return n_lists


def test_caps_and_suppression_policies():
    assert ps.largest_cap(6000) == 2774 and ps.largest_cap(8192) == 801 and ps.largest_cap(1815) == 4096
    assert ps.lists_fit(6000, 2774) and not ps.lists_fit(1815, ps.LIST_MIN_DET) and not ps.lists_fit(2048, ps.LIST_MIN_DET)
    n = run_caps_and_policy()
    assert n >= 12


def test_caps_reached_inside_a_chunk():
    """Small, far-apart boxes: (almost) nothing is suppressed, so the cap is reached at a chosen place inside a 64-candidate
    chunk -- in its lower and upper 32-candidate halves, at its end and one past it."""
    d = ps.random_dets(111, 2, 2048, side=640.0, size=2.0)
    for md in (1, 2, 31, 32, 33, 40, 63, 64, 65, 96, 127, 128, 129, 300, 301):
        counts = check_nms(d, 0.001, 0.45, md)
        assert counts.tolist() == [md, md]


def test_largest_cap_that_fits_and_the_next_is_refused():
    d = ps.random_dets(112, 1, ps.MAX_CAND, side=640.0, size=12.0)
    counts = check_nms(d, 0.001, 0.45, 801)
    assert int(counts[0]) == 801
    with pytest.raises(eng.Yfv2Error, match="shared memory"):
        eng.nms(torch.from_numpy(d).cuda(), 0.001, 0.45, max_det=802)


# ---------------------------------------------------------------------------------------------------------------------------
# sort sizes

NMS_CNTS = [1, 63, 64, 65, 128, 255, 256, 257, 512, 1024, 1025, 2048, 2049, 4096, 8192]


def run_nms_sort_sizes(cnts=NMS_CNTS):
    for k, cnt in enumerate(cnts):
        M = min(ps.MAX_CAND, cnt + 37 * (k + 1))
        d = ps.random_dets(120 + k, 1, M, side=640.0, size=40.0, n_pass=cnt)
        assert len(ps.candidates(d[0], 0.001)[0]) == cnt
        check_nms(d, 0.001, 0.45, min(4096, ps.largest_cap(M)))


def test_nms_sort_sizes():
    assert sorted(set(ps.sort_size(c) for c in NMS_CNTS)) == [64, 128, 256, 512, 1024, 2048, 4096, 8192]
    run_nms_sort_sizes()


def fused_sort_case(seed, cnt, H, W, A, C):
    """Head logits with exactly `cnt` (cell, anchor) pairs above conf_thres = 1e-3: their objectness logit is +8 (sigmoid > 0.999,
    times a softmax maximum >= 1/C), every other one -30."""
    hs = heads(seed, 1, H, W, A, C)
    rs = np.random.RandomState(seed)
    sizes = [hs[1].size, hs[4].size]
    on = np.zeros(sum(sizes), bool)
    on[rs.permutation(len(on))[:cnt]] = True
    hs[1] = np.where(on[:sizes[0]].reshape(hs[1].shape), 8.0, -30.0).astype(np.float32)
    hs[4] = np.where(on[sizes[0]:].reshape(hs[4].shape), 8.0, -30.0).astype(np.float32)
    return hs


def profiled_candidates(preds, cfg, ct, it, max_det):
    """Candidate counts the fused kernel reports in slot 9 of yfv2_debug_nms_profile, and its outputs in that mode."""
    buf = torch.zeros(preds[0].shape[0], 16, dtype=torch.int64, device="cuda")
    assert eng.lib().yfv2_debug_nms_profile(ctypes.c_void_p(buf.data_ptr())) == 0
    try:
        res = eng.decode_nms(preds, cfg, ct, it, max_det=max_det, want_idx=True)
        torch.cuda.synchronize()
    finally:
        eng.lib().yfv2_debug_nms_profile(None)
    return buf[:, 9].cpu().numpy(), res


FUSED_CNTS = [(64, 640, 640, 3, 80), (65, 640, 640, 3, 80), (256, 640, 640, 3, 80), (257, 640, 640, 3, 80),
              (1024, 640, 640, 3, 80), (2048, 640, 640, 3, 80), (2049, 640, 640, 3, 80), (4096, 640, 640, 3, 80),
              (2048, 384, 544, 8, 20), (8160, 384, 544, 8, 20)]


def run_fused_sort_sizes(cases=FUSED_CNTS, warp_cells=False):
    for k, (cnt, H, W, A, C) in enumerate(cases):
        hs = to_dev(fused_sort_case(130 + k, cnt, H, W, A, C))
        cfg = cfg_for(A, C, H, W)
        M = (H * W // 256 + H * W // 1024) * A
        # the warp-per-cell path stages the logits of 32 cells behind the NMS state
        md = min(4096, ps.largest_cap(M, (5 * A + C) * 33 * 4 if warp_cells or C > 80 else 0))
        dh, counts = check_fused(hs, cfg, 0.001, 0.45, md)
        assert len(ps.candidates(dh[0], 0.001)[0]) == cnt
        pc, (p_out, p_counts, p_idx) = profiled_candidates(hs, cfg, 0.001, 0.45, md)
        assert pc.tolist() == [cnt], (cnt, H, W, A, C)
        f_out, f_counts, f_idx = eng.decode_nms(hs, cfg, 0.001, 0.45, max_det=md, want_idx=True)
        assert torch.equal(p_out, f_out) and torch.equal(p_counts, f_counts) and torch.equal(p_idx, f_idx)


def test_fused_sort_sizes():
    run_fused_sort_sizes()


# ---------------------------------------------------------------------------------------------------------------------------
# rounding edges

def run_near_midpoint_pairs(thrs=(0.3, 0.4, 0.45, 0.5), caps=(300,)):
    outcomes = set()
    for k, thr in enumerate(thrs):
        a, b, above, rel = ps.near_mid_pairs(thr, 20, 140 + k, min_side=400)
        assert rel.max() < 1e-6 and above.sum() == 20 and (~above).sum() == 20
        for layout in ("adjacent", "split"):
            d = np.stack([ps.pair_image(a[:40], b[:40], layout)])
            for md in caps:
                check_nms(d, 0.001, thr, md)
        rows, _ = opost.nms(torch.from_numpy(ps.pair_image(a, b, "adjacent")[None]), 0.001, thr, return_indices=True)
        outcomes.add((thr, rows[0].shape[0] < 80))
        outcomes.add((thr, rows[0].shape[0] > 40))
    return outcomes


def test_iou_within_1e6_of_the_rounding_boundary():
    """Integer-corner pairs whose IoU lies within 1e-6 of the boundary, on both sides: the fp32 pre-test must hand them to the
    exact fp64 test, inside one chunk and against the kept list."""
    outcomes = run_near_midpoint_pairs()
    assert all(v for _, v in outcomes)                                       # each threshold suppresses some pairs, keeps others


def run_zone_pairs(thrs=(0.3, 0.35, 0.4)):
    for k, thr in enumerate(thrs):
        for layout in ("adjacent", "split"):
            d, sup = ps.zone_image(thr, 16, 150 + k, layout)
            counts = check_nms(d[None], 0.001, thr, 300)
            assert int(counts[0]) == 64 + int((~sup).sum())


def test_iou_between_the_boundary_and_its_fp32_rounding():
    """Pairs an fp32 estimate of the boundary alone gets wrong; the 1e-6 guard band of iou_fast must route them to iou_gt."""
    for thr in (0.3, 0.35, 0.4):
        assert len(ps.zone_heights(thr, 16, 0)[0]) == 16
    run_zone_pairs()


def test_iou_exactly_at_the_threshold():
    """IoU exactly at the threshold: 1/2 at 0.5 is kept (fl32(0.5) is not above 0.5); 2/5 at 0.4 is suppressed (fl32(0.4) is
    above 0.4 as a double); 9/20 at 0.45 is kept (fl32(0.45) is below 0.45)."""
    a = np.array([[0, 0, 3, 1], [10, 0, 15, 2], [20, 0, 30, 10], [40, 0, 45, 4]], np.float64)
    b = np.array([[1, 0, 4, 1], [10, 0, 12, 2], [20, 0, 30, 5], [40, 0, 43, 3]], np.float64)
    # IoU 2/4, 4/10 (b inside a), 50/100, 9/20
    d = np.stack([ps.pair_image(a, b, "adjacent")])
    assert check_nms(d, 0.001, 0.5).tolist() == [8]
    assert check_nms(d, 0.001, 0.45).tolist() == [4 + 2]                   # 0.5 and 0.5 suppressed; 0.4 and 0.45 kept
    assert check_nms(d, 0.001, 0.4).tolist() == [4]                        # 0.4 exactly suppressed too


def test_thresholds_outside_the_open_unit_interval():
    d = ps.random_dets(160, 2, 1815, side=352.0)
    dg = np.stack([ps.degenerate_image(161), ps.degenerate_image(162)])
    for it in (-0.1, 0.0, 1.0, 1.5):
        for md in (300, 1000):
            check_nms(d, 0.001, it, md)
            check_nms(dg, 0.3, it, md)
    assert check_nms(d, 0.001, -0.1).tolist() == [1, 1]                    # every IoU (0 included) is above -0.1


def test_degenerate_boxes_raw():
    dg = np.stack([ps.degenerate_image(170 + k) for k in range(4)])
    for it in (0.3, 0.45, 0.5):
        for ct in (0.001, 0.4):
            for wh in (4096.0, 0.0):
                check_nms(dg, ct, it, 300, wh)


def test_score_ties_at_a_chunk_boundary_and_at_the_cap():
    d = np.stack([ps.tie_image(180), ps.tie_image(181)])
    for md in (300, 310, 1000):
        check_nms(d, 0.001, 0.45, md)
    counts = check_nms(d, 0.001, 0.45, 300)
    assert counts.tolist() == [300, 300]


# ---------------------------------------------------------------------------------------------------------------------------
# fused candidate generation

FUSED_SHAPES = [(3, 80), (2, 80), (8, 20), (1, 1), (3, 81), (3, 256)]


def tie_heads(seed, n, H, W, A, C):
    """Class logits with exact ties of the maximum and ties a few ulps apart, on a third of the cells each."""
    hs = heads(seed, n, H, W, A, C)
    rs = np.random.RandomState(seed)
    for lv in (2, 5):
        cl = hs[lv]
        if C < 3:
            continue
        n_, _, h, w = cl.shape
        for i in range(n_):
            for y in range(h):
                for x in range(w):
                    r = rs.randint(3)
                    cs = rs.choice(C, 3, replace=False)
                    v = np.float32(6.0 + rs.rand())
                    if r == 0:
                        cl[i, cs, y, x] = v                                              # exact ties
                    elif r == 1:
                        steps = rs.randint(0, 4, 3).astype(np.int32)
                        cl[i, cs, y, x] = (np.full(3, v).view(np.int32) + steps).view(np.float32)   # a few ulps apart
    return hs


def subnormal_heads(seed, n, H, W, A, C):
    """Objectness logits in [-89, -87] (sigmoid 0 .. 1.6e-38: products with the class probability are subnormal) and class
    logits within 1e-3 of each other, so that classes further than 1e-5 below the maximum round to the same product."""
    hs = heads(seed, n, H, W, A, C)
    rs = np.random.RandomState(seed)
    for lv in (1, 4):
        hs[lv] = rs.uniform(-89.0, -87.0, hs[lv].shape).astype(np.float32)
    for lv in (2, 5):
        hs[lv] = (rs.rand(*hs[lv].shape) * rs.choice([1e-5, 1e-4, 1e-3], hs[lv].shape)).astype(np.float32)
    return hs


def run_fused_shapes(shapes=FUSED_SHAPES, H=352, W=352):
    for k, (A, C) in enumerate(shapes):
        cfg = cfg_for(A, C, H, W)
        hs = to_dev(heads(190 + k, 2, H, W, A, C))
        for ct, it in ((0.001, 0.45), (0.3, 0.5)):
            for md in (300, 1000):
                check_fused(hs, cfg, ct, it, md)


def test_fused_shapes():
    run_fused_shapes()


def run_fused_ties(shapes=((3, 80), (2, 80), (8, 20), (3, 81))):
    for k, (A, C) in enumerate(shapes):
        cfg = cfg_for(A, C, 224, 224)
        check_fused(to_dev(tie_heads(200 + k, 2, 224, 224, A, C)), cfg, 0.001, 0.45)


def test_fused_class_ties():
    run_fused_ties()


def run_fused_subnormal(shapes=((3, 80), (2, 80), (8, 20), (3, 81))):
    for k, (A, C) in enumerate(shapes):
        cfg = cfg_for(A, C, 352, 352)
        dh, counts = check_fused(to_dev(subnormal_heads(210 + k, 2, 352, 352, A, C)), cfg, 0.0, 0.45, 1000)
        assert int(counts.min()) > 0
        conf = ps.candidates(dh[0], 0.0)[1]
        assert len(conf) and conf.max() < np.finfo(np.float32).tiny


def test_fused_subnormal_confidences():
    """conf = p * obj below FLT_MIN carries fewer than 24 bits: a class far more than 1e-5 below the maximum can round to the
    same product, and the reference then reports the first such class."""
    run_fused_subnormal()


# ---------------------------------------------------------------------------------------------------------------------------
# runtime switches: read once per process, so each runs in a child

SWITCH_RUNS = {
    "YFV2_NMS_WARP_PER_CELL": "T.run_fused_shapes([(3, 80), (2, 80), (8, 20)]); T.run_fused_ties(); T.run_fused_subnormal(); "
                              "T.run_fused_sort_sizes(T.FUSED_CNTS[6:], warp_cells=True)",
    "YFV2_NMS_LISTS": "assert T.run_caps_and_policy(True, ['m1815', 'm2048', 'm6000_640'], [64, 65, 300, 338]) >= 4; "
                      "T.run_near_midpoint_pairs(caps=(64, 300)); T.run_zone_pairs(); T.run_fused_subnormal([(3, 80), (8, 20)])",
}


@pytest.mark.parametrize("switch", list(SWITCH_RUNS))
def test_runtime_switch(switch):
    code = "import sys; sys.path[:0] = [%r, %r]; import test_post_space_gpu as T; %s; print('ok')" % (
        ROOT, os.path.join(ROOT, "tests"), SWITCH_RUNS[switch])
    env = dict(os.environ, **{switch: "1"})
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=ROOT, timeout=600)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stderr[-3000:]

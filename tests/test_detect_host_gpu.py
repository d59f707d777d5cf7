"""yfv2_detect_u8_host, the whole evaluation step from host uint8 images to host detections, against a chain of trusted oracles:
its rows [:count] and counts equal yfv2_decode_nms(forward_u8(x)) on the same plan bit for bit, those rows equal oracle.post.nms
on the device-decoded candidates bit for bit, and at the benchmark geometry forward_u8's head tensors match the fp64 oracle
forward.  Shapes reach every decode+NMS kernel variant and both head kernels; thresholds reach the max_det cap and empty results;
the benchmark's three plans on three streams must give what one stream gives.  Requests the fused decode+NMS refuses, and buffers
that do not fit the plan, are refused before anything is enqueued: the workspace and the host buffers keep a sentinel.
Rows past a count are unspecified and never compared."""
import ctypes

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import post_space as ps
import synth
from oracle import net as onet, post as opost
from test_forward_fp64_gpu import E2E_BOUND, nerr

pytestmark = pytest.mark.gpu


def cfg_for(H, W, A, C):
    c = synth.coco_cfg(W, H, C)
    c["anchor_num"], c["anchors"] = A, list(synth.COCO_ANCHORS[:4 * A])
    return c


class Net:
    """A packed plan with its weights (the weight tensors stay alive as long as the plan)."""

    def __init__(self, N, H, W, A, C, sd, detect_max_det):
        import yfv2_engine as eng
        import model.detector as det
        self.m = det.Detector(C, A, True)
        self.m.load_state_dict(sd, strict=True)
        self.m = self.m.cuda().eval()
        self.plan = eng.Plan("cuda", N, H, W, A, C, detect_max_det=detect_max_det)
        self.keep = self.plan.pack(*self.m._weight_tensors())
        self.cfg = cfg_for(H, W, A, C)
        self.anchors = eng.anchors_array(self.cfg)


def host_buffers(N, max_det):
    return torch.empty((N, max_det, 6), dtype=torch.float32).pin_memory(), torch.empty((N,), dtype=torch.int32).pin_memory()


def detect_host(net, x_u8, conf, iou, max_det):
    out, cnt = host_buffers(x_u8.shape[0], max_det)
    net.plan.detect_u8_host(x_u8.contiguous().pin_memory(), net.anchors, conf, iou, out, cnt, max_det)
    torch.cuda.synchronize()
    return out, cnt


def check_against_chain(net, x_u8, conf, iou, max_det, got=None):
    """detect_u8_host == decode_nms(forward_u8) on the same plan, and those rows == oracle.post.nms(decode(preds))."""
    import yfv2_engine as eng
    out, cnt = got if got is not None else detect_host(net, x_u8, conf, iou, max_det)
    preds = net.plan.forward(x_u8.cuda())
    ref, ref_cnt, _ = eng.decode_nms(preds, net.cfg, conf, iou, max_det=max_det)
    ref, ref_cnt = ref.cpu(), ref_cnt.cpu()
    assert torch.equal(cnt, ref_cnt), (cnt, ref_cnt)
    for i, k in enumerate(cnt.tolist()):
        assert 0 <= k <= max_det
        assert torch.equal(out[i, :k], ref[i, :k]), i
    want = opost.nms(eng.decode(preds, net.cfg).cpu(), conf, iou, max_det=max_det)
    for i, w in enumerate(want):
        k = int(ref_cnt[i])
        assert k == w.shape[0] and np.array_equal(ref[i, :k].numpy(), w.numpy()), i
    return preds, cnt


def u8_images(seed, N, H, W):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(N, 3, H, W, generator=g) * 255).to(torch.uint8)


# ---- the benchmark geometry ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def bench_net():
    import bench
    _, sd = bench.random_state_dict()
    return Net(bench.BATCH, bench.SIDE, bench.SIDE, bench.ANCHORS, bench.CLASSES, sd, 300), sd


def test_bench_geometry(bench_net):
    """N=256 at 352^2, A=3, C=80, conf 0.001, IoU 0.4, max_det 300 (decode_nms_kernel<..., 2>); the u8 head tensors of images
    0, 127 and 255 against the fp64 oracle forward of x / 255."""
    import bench
    net, sd = bench_net
    x = u8_images(11, bench.BATCH, bench.SIDE, bench.SIDE)
    preds, cnt = check_against_chain(net, x, bench.CONF, bench.IOU, 300)
    assert int(cnt.sum()) > 0
    idx = [0, 127, 255]
    sd64 = {k: v.double() if v.is_floating_point() else v for k, v in sd.items()}
    with torch.no_grad():
        ref = onet.forward(sd64, x[idx].double() / 255)
    err = max(nerr(p[idx].double().cpu(), r) for p, r in zip(preds, ref))
    print("\nuint8 end to end, bench weights: %.3e" % err)
    assert err <= E2E_BOUND, err


def test_bench_e2e_pattern_matches_one_stream(bench_net):
    """bench.py's e2e leg: 3 plans built with detect_max_det=300 on 3 streams, 6 steps rotated i % 3, each step with its own
    pinned input and output buffers; after one synchronise every step's result equals a single-stream run on a fresh plan."""
    import bench
    import yfv2_engine as eng
    net, sd = bench_net
    B, S = bench.BATCH, bench.SIDE
    nets = [Net(B, S, S, bench.ANCHORS, bench.CLASSES, sd, eng.MAX_DET) for _ in range(3)]
    streams = [torch.cuda.Stream() for _ in range(3)]
    xs = [u8_images(20 + i, B, S, S).pin_memory() for i in range(6)]
    bufs = [host_buffers(B, eng.MAX_DET) for _ in range(6)]
    torch.cuda.synchronize()
    for i in range(6):
        with torch.cuda.stream(streams[i % 3]):
            nets[i % 3].plan.detect_u8_host(xs[i], nets[i % 3].anchors, bench.CONF, bench.IOU, bufs[i][0], bufs[i][1])
    torch.cuda.synchronize()
    del nets
    fresh = Net(B, S, S, bench.ANCHORS, bench.CLASSES, sd, eng.MAX_DET)
    for i in range(6):
        out, cnt = detect_host(fresh, xs[i], bench.CONF, bench.IOU, eng.MAX_DET)
        assert torch.equal(bufs[i][1], cnt), i
        for n, k in enumerate(cnt.tolist()):
            assert torch.equal(bufs[i][0][n, :k], out[n, :k]), (i, n)


# ---- trained weights on real photographs -----------------------------------------------------------------------------------
@pytest.mark.parametrize("conf,iou", [(0.01, 0.4), (0.3, 0.4)])
def test_modelzoo_photos(golden_dir, conf, iou):
    import os
    import yfv2_engine as eng
    import resize_cases as rc
    w = synth.load_modelzoo_weights(golden_dir)
    net = Net(2, 352, 352, 3, 80, {k: torch.from_numpy(v) for k, v in w.items()}, 300)
    frames = np.load(os.path.join(golden_dir, "frames_modelzoo.npz"))
    x = eng.resize_bgr([frames[n] for n in rc.MODELZOO_FRAMES], 352, 352).cpu()
    _, cnt = check_against_chain(net, x, conf, iou, 300)
    assert cnt.min() >= 1, cnt


# ---- other shapes: every decode+NMS variant, both head kernels, the largest candidate count ---------------------------------
SHAPES = {   # name -> (N, H, W, A, C, max_det)
    "1x32x32_md1": (1, 32, 32, 3, 80, 1),
    "3x96x160_a2c20_md7": (3, 96, 160, 2, 20, 7),         # decode_nms_kernel variant 1
    "2x96x128_c150": (2, 96, 128, 3, 150, 300),           # variant 0 (warp per cell) and head2_kernel
    "5x224x96": (5, 224, 96, 3, 80, 300),
    "2x736_largest_cap": (2, 736, 736, 3, 80, None),      # M = 7935 <= 8192, the largest max_det whose NMS state fits
}


@pytest.mark.parametrize("name", list(SHAPES))
def test_shapes(name):
    N, H, W, A, C, md = SHAPES[name]
    if md is None:
        M = A * ((H // 16) * (W // 16) + (H // 32) * (W // 32))
        assert M == 7935
        md = ps.largest_cap(M)
    sd = synth.make_state_dict(300 + len(name), classes=C, anchor_num=A)
    net = Net(N, H, W, A, C, sd, md)
    check_against_chain(net, u8_images(len(name), N, H, W), 0.001, 0.4, md)


@pytest.mark.parametrize("conf,iou", [(0.0, 0.4), (1.0, 0.4), (0.001, 0.0), (0.001, 1.0)])
def test_thresholds(conf, iou):
    net = Net(5, 224, 96, 3, 80, synth.make_state_dict(310), 300)
    _, cnt = check_against_chain(net, u8_images(31, 5, 224, 96), conf, iou, 50)
    if conf == 0.0:
        assert (cnt == 50).all(), cnt                    # every candidate passes: each image hits the cap
    if conf == 1.0:
        assert (cnt == 0).all(), cnt                     # no score exceeds 1


def test_forward_around_detect_is_unchanged():
    """forward() on float input, then detect_u8_host, then forward() again on the same plan: both forwards are bit-identical."""
    net = Net(3, 96, 128, 3, 80, synth.make_state_dict(320), 300)
    xf = synth.make_images(321, 3, 96, 128).cuda()
    first = [p.clone() for p in net.plan.forward(xf)]
    check_against_chain(net, u8_images(322, 3, 96, 128), 0.01, 0.4, 300)
    second = net.plan.forward(xf)
    for a, b in zip(first, second):
        assert torch.equal(a, b)


# ---- refusals before anything is enqueued -----------------------------------------------------------------------------------
SENTINEL = 0xA5


def refusals(net, N, H, W, A, md):
    """(label, call) pairs that must raise; x, out, counts are the valid buffers for max_det md."""
    x = u8_images(40, N, H, W).pin_memory()
    out, cnt = host_buffers(N, md)

    def call(x_=x, out_=out, cnt_=cnt, max_det=md, anchors=None):
        return lambda: net.plan.detect_u8_host(x_, anchors if anchors is not None else net.anchors, 0.01, 0.4, out_, cnt_, max_det)
    few = (ctypes.c_double * (4 * A - 1))(*synth.COCO_ANCHORS[:4 * A - 1])
    return x, out, cnt, [
        ("x shape", call(x_=u8_images(41, N, H, W + 32).pin_memory())),
        ("x dtype", call(x_=x.float())),
        ("x on cuda", call(x_=x.cuda())),
        ("out shape", call(out_=host_buffers(N, md + 1)[0])),
        ("out dtype", call(out_=out.double())),
        ("counts shape", call(cnt_=host_buffers(N + 1, md)[1])),
        ("counts dtype", call(cnt_=cnt.long())),
        ("too few anchors", call(anchors=few)),
    ]


def expect_refused(net, calls, host):
    import yfv2_engine as eng
    net.plan.workspace.fill_(SENTINEL)
    for t in host:
        t.view(torch.uint8).fill_(SENTINEL)
    torch.cuda.synchronize()
    for label, fn in calls:
        with pytest.raises(eng.Yfv2Error):
            fn()
        torch.cuda.synchronize()
        assert bool((net.plan.workspace == SENTINEL).all()), label
        for t in host:
            assert bool((t.view(torch.uint8) == SENTINEL).all()), label


def test_refused_before_anything_is_enqueued():
    N, H, W, A, C = 2, 64, 96, 3, 80
    sd = synth.make_state_dict(330)
    sized = Net(N, H, W, A, C, sd, 300)
    x, out, cnt, calls = refusals(sized, N, H, W, A, 300)
    import yfv2_engine as eng
    over = 301                                   # the smallest max_det whose buffers no longer fit (the layout pads to 256 bytes)
    while eng.lib().yfv2_detect_workspace_bytes(sized.plan._h, over) <= sized.plan.workspace.numel():
        over += 1
    calls += [("max_det 0", lambda: sized.plan.detect_u8_host(x, sized.anchors, 0.01, 0.4, host_buffers(N, 0)[0], cnt, 0)),
              ("max_det above the plan's sizing",
               lambda: sized.plan.detect_u8_host(x, sized.anchors, 0.01, 0.4, host_buffers(N, over)[0], cnt, over))]
    expect_refused(sized, calls, [out, cnt])
    check_against_chain(sized, x, 0.01, 0.4, 300)

    unsized = Net(N, H, W, A, C, sd, 0)          # detect_max_det=0: the workspace holds the forward only
    x, out, cnt, _ = refusals(unsized, N, H, W, A, 300)
    expect_refused(unsized, [("detect_max_det=0", lambda: unsized.plan.detect_u8_host(x, unsized.anchors, 0.01, 0.4, out, cnt))],
                   [out, cnt])

    big = Net(N, H, W, A, C, sd, 4097)           # sized for 4097 rows: the NMS's own limit refuses
    out4097, _ = host_buffers(N, 4097)
    expect_refused(big, [("max_det 4097", lambda: big.plan.detect_u8_host(x, big.anchors, 0.01, 0.4, out4097, cnt, 4097))],
                   [out4097, cnt])
    check_against_chain(big, x, 0.01, 0.4, 300)


def test_too_many_candidates_refused_before_anything_is_enqueued():
    """A 1024^2 plan has 15360 candidates per image, more than the NMS takes: refused before the copy and the forward."""
    import yfv2_engine as eng
    net = Net(1, 1024, 1024, 3, 80, synth.make_state_dict(340), 300)
    x = u8_images(41, 1, 1024, 1024).pin_memory()
    out, cnt = host_buffers(1, 300)
    expect_refused(net, [("1024^2", lambda: net.plan.detect_u8_host(x, net.anchors, 0.01, 0.4, out, cnt))], [out, cnt])
    with pytest.raises(eng.Yfv2Error, match="M=15360 candidates per image exceeds 8192"):
        net.plan.detect_u8_host(x, net.anchors, 0.01, 0.4, out, cnt)

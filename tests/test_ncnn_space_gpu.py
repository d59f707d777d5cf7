"""GPU: the deploy post-process (yfv2_ncnn_post) across anchors, classes, shapes, thresholds and limits (tests/ncnn_space.py),
bit for bit against the reference's own C++ (tests/golden/ncnn_space.npz) and oracle/ncnn_post.c; the raw output buffers past
the kept rows; batches against images run alone; and yfv2_export_heads against an fp64 sigmoid | sigmoid | softmax."""
import ctypes

import numpy as np
import pytest
import torch

import ncnn_space as ns
from test_ncnn_space_cpu import CASES, GOLDEN, run_oracle

pytestmark = pytest.mark.gpu
f32 = np.float32


def _eng():
    import yfv2  # noqa: F401
    import yfv2_engine
    return yfv2_engine


def run_device(c, N=1, max_out=None):
    eng = _eng()
    o2 = torch.from_numpy(np.ascontiguousarray(c["out2"]))[None].expand(N, -1, -1, -1).contiguous().cuda()
    o3 = torch.from_numpy(np.ascontiguousarray(c["out3"]))[None].expand(N, -1, -1, -1).contiguous().cuda()
    return eng.ncnn_post(o2, o3, c["A"], float(c["thresh"]), float(c["nms"]), c["src"], anchors=[float(a) for a in c["anchors"]],
                         max_out=max_out)


def same(got, want):
    b, s, k = got
    wb, ws, wk = want
    assert len(s) == len(ws), (len(s), len(ws))
    assert np.array_equal(b, wb) and np.array_equal(k, wk)
    assert np.array_equal(np.asarray(s, f32).view(np.uint32), np.asarray(ws, f32).view(np.uint32))


@pytest.mark.parametrize("name", sorted(CASES))
def test_matches_the_reference_and_the_oracle(name):
    """Every case: the device equals the oracle, and the reference's own outputs where they are frozen (all cases but those with
    equal scores among more than 16 candidates, whose order the reference leaves to introsort)."""
    c = GOLDEN.get(name, CASES[name])
    (got,) = run_device(c)
    same(got, run_oracle(c))
    if name in GOLDEN:
        same(got, (c["boxes"], c["scores"], c["cates"]))


def _raw(c, N, max_out):
    """yfv2_ncnn_post through the C ABI into buffers pre-filled with a pattern: (boxes, scores, cates, counts) as numpy."""
    eng = _eng()
    o2 = torch.from_numpy(np.ascontiguousarray(c["out2"]))[None].expand(N, -1, -1, -1).contiguous().cuda()
    o3 = torch.from_numpy(np.ascontiguousarray(c["out3"]))[None].expand(N, -1, -1, -1).contiguous().cuda()
    boxes = torch.full((N, max_out, 4), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
    scores = torch.full((N, max_out), 7.5, dtype=torch.float32, device="cuda")
    cates = torch.full((N, max_out), 0x5A5A, dtype=torch.int32, device="cuda")
    counts = torch.full((N,), -7, dtype=torch.int32, device="cuda")
    sw, sh = ns.scales(c)
    anc = (ctypes.c_float * (4 * c["A"]))(*[float(a) for a in c["anchors"]])
    p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    rc = eng.lib().yfv2_ncnn_post(p(o2), p(o3), N, c["H"], c["W"], c["A"], c["C"], anc, ctypes.c_float(c["thresh"]),
                                  ctypes.c_float(c["nms"]), ctypes.c_float(sw), ctypes.c_float(sh), max_out, p(boxes), p(scores),
                                  p(cates), p(counts), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0
    torch.cuda.synchronize()
    return boxes.cpu().numpy(), scores.cpu().numpy(), cates.cpu().numpy(), counts.cpu().numpy()


@pytest.mark.parametrize("name", ["max_out", "chunk_129", "thr_one", "limit_a3_672"])
def test_max_out_edges_padding_and_counts(name):
    """max_out 1, count-1, count, count+1 (and 2*count + 3): rows past min(count, max_out) are zero with cate -1 in the raw
    buffers, the first rows are the untruncated result's, and counts reports the untruncated count."""
    c = GOLDEN[name]
    want = (c["boxes"], c["scores"], c["cates"])
    n = len(want[1])
    for max_out in sorted({m for m in ns.max_out_edges(n) + [2 * n + 3] if m >= 1}):
        b, s, k, cnt = _raw(c, 2, max_out)
        r = min(n, max_out)
        for i in range(2):
            assert cnt[i] == n
            same((b[i, :r], s[i, :r], k[i, :r]), (want[0][:r], want[1][:r], want[2][:r]))
            assert (b[i, r:] == 0).all() and (s[i, r:] == 0).all() and (k[i, r:] == -1).all(), (name, max_out)


@pytest.mark.parametrize("N", [1, 7, 512])
def test_batch_equals_each_image_alone(N):
    """N images in one launch (one CTA per image): each equals the same image run alone, and the oracle."""
    pool = [c for c in CASES.values() if (c["A"], c["C"], c["H"], c["W"]) == (3, 80, 64, 160)]
    rs = np.random.RandomState(N)
    pool += [ns.random_head("batch%d" % i, 1000 + i, 3, 80, 64, 160, classes=2) for i in range(16 - len(pool))]
    pick = rs.randint(len(pool), size=N)
    o2 = torch.from_numpy(np.stack([pool[i]["out2"] for i in pick])).cuda()
    o3 = torch.from_numpy(np.stack([pool[i]["out3"] for i in pick])).cuda()
    c0 = pool[0]
    eng = _eng()
    anc = [float(a) for a in c0["anchors"]]
    res = eng.ncnn_post(o2, o3, 3, float(c0["thresh"]), float(c0["nms"]), c0["src"], anchors=anc)
    alone = {}
    for j, i in enumerate(pick):
        if i not in alone:
            c = dict(pool[i], anchors=c0["anchors"], thresh=c0["thresh"], nms=c0["nms"], src=c0["src"])
            (alone[i],) = run_device(c)
            same(alone[i], run_oracle(c))
        same(res[j], alone[i])
    assert sum(len(r[1]) for r in res) > 10 * N


def _fp64_export(preds):
    outs = []
    for lv in range(2):
        reg, obj, cls = [p.double() for p in preds[3 * lv:3 * lv + 3]]
        o = torch.cat((torch.sigmoid(reg), torch.sigmoid(obj), torch.softmax(cls, 1)), 1).permute(0, 2, 3, 1)
        outs.append(o.contiguous())
    return outs


EXPORT_BOUND = 2.0 ** -21          # absolute, on values in [0, 1]


def _export_logits(seed, A, C, N=2, H=64, W=96):
    rs = np.random.RandomState(seed)
    preds = []
    for lv, s in enumerate((16, 32)):
        h, w = H // s, W // s
        reg = rs.normal(0, 4, (N, 4 * A, h, w))
        obj = rs.normal(0, 4, (N, A, h, w))
        cls = rs.normal(0, 6, (N, C, h, w))
        reg[0, :, 0, 0] = 100.0; reg[0, :, 0, 1] = -100.0                 # saturated sigmoids
        obj[0, :, 0, 0] = 100.0; obj[1, :, 0, 0] = -100.0
        cls[0, :, 0, 0] = 3.25                                            # all-equal class logits: exactly 1/C each
        if h * w > 1:
            cls[0, :, 0, 1] = -100.0; cls[0, C // 2, 0, 1] = 100.0       # one dominant logit
            cls[1, :, 0, 1] = 100.0                                       # all at +100
        preds += [reg, obj, cls]
    return [torch.from_numpy(p.astype(f32)) for p in preds]


@pytest.mark.parametrize("A", [1, 3, 8])
@pytest.mark.parametrize("C", [1, 31, 32, 33, 150, 256])
def test_export_heads_against_fp64(A, C):
    """export_heads within EXPORT_BOUND = 2^-21 = 4.8e-7 (absolute; every output lies in [0, 1]) of sigmoid | sigmoid | softmax
    in fp64 of the same fp32 logits, channel-last; logits of +-100, all-equal class logits and one dominant logit included.
    Measured worst case over the 18 shapes: 2.16e-7 (A=1, C=256) on an H100 80GB HBM3 at 700 W, under 4 fp32 ulps of 1."""
    eng = _eng()
    preds = _export_logits(10 * A + C, A, C)
    o2, o3 = eng.export_heads([p.cuda() for p in preds])
    w2, w3 = _fp64_export(preds)
    worst = 0.0
    for got, want in ((o2, w2), (o3, w3)):
        assert got.shape == want.shape and got.dtype == torch.float32
        g = got.cpu().double()
        assert torch.isfinite(g).all()
        worst = max(worst, float((g - want).abs().max()))
    assert worst <= EXPORT_BOUND, worst


@pytest.mark.parametrize("A,C", [(1, 1), (1, 31), (3, 32), (3, 33), (8, 150), (3, 150), (8, 1)])
def test_export_heads_equals_the_export_onnx_detector(A, C):
    """Detector(export_onnx=True) returns export_heads of the plain Detector's heads, bit for bit (A + C <= 192: the heads'
    output convolution limit)."""
    eng = _eng()
    import synth
    import model.detector as det
    sd = synth.make_state_dict(A * 1000 + C, classes=C, anchor_num=A)
    x = synth.make_images(A + C, 2, 64, 96).cuda()
    m = det.Detector(C, A, True).cuda().eval()
    m.load_state_dict(sd)
    e = det.Detector(C, A, True, True).cuda().eval()
    e.load_state_dict(sd)
    with torch.no_grad():
        preds = m(x)
        o2, o3 = eng.export_heads(preds)
        g2, g3 = e(x)
    assert torch.equal(o2, g2) and torch.equal(o3, g3)
    assert o2.shape == (2, 4, 6, 5 * A + C) and o3.shape == (2, 2, 3, 5 * A + C)


class _NoLib:
    def __getattr__(self, name):
        raise AssertionError("the library was called (%s) with tensors that do not fit together" % name)


def test_mismatched_tensors_are_refused_before_the_library(monkeypatch):
    """Device tensors whose shapes disagree: every wrapper raises Yfv2Error naming the tensor and the expected shape, and never
    reaches the library (replaced by a stub that fails the test)."""
    eng = _eng()
    monkeypatch.setattr(eng, "lib", lambda: _NoLib())
    d = "cuda"
    o2 = torch.zeros(2, 4, 6, 95, device=d)
    for s3 in ((2, 1, 3, 95), (2, 2, 2, 95), (2, 2, 3, 94), (1, 2, 3, 95), (3, 2, 3, 95)):
        with pytest.raises(eng.Yfv2Error, match="out3 has shape"):
            eng.ncnn_post(o2, torch.zeros(s3, device=d), 3)
    with pytest.raises(eng.Yfv2Error, match="out3"):
        eng.ncnn_post(o2, torch.zeros(2, 2, 3, 95), 3)                       # on the CPU
    A, C = 3, 80
    good = [(2, 4 * A, 4, 6), (2, A, 4, 6), (2, C, 4, 6), (2, 4 * A, 2, 3), (2, A, 2, 3), (2, C, 2, 3)]
    cfg = {"height": 64, "width": 96, "anchors": [1.0] * 4 * A}
    for i in range(6):
        for dim in range(4):
            shape = [list(s) for s in good]
            shape[i][dim] -= 1
            preds = [torch.zeros(s, device=d) for s in shape]
            for fn in (eng.export_heads, lambda p: eng.decode(p, cfg), lambda p: eng.decode_nms(p, cfg)):
                with pytest.raises(eng.Yfv2Error, match="preds"):
                    fn(preds)
    preds = [torch.zeros(s, device=d) for s in good]
    preds[4] = preds[4].cpu()
    with pytest.raises(eng.Yfv2Error, match=r"preds\[4\]"):
        eng.export_heads(preds)

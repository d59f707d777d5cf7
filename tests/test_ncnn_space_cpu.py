"""CPU side of the deploy post-process's parameter space (tests/ncnn_space.py): oracle/ncnn_post.c against the outputs of the
reference's own C++ (tests/golden/ncnn_space.npz, make_golden_ncnn_space.py) bit for bit, every case on the side it was built
for, push order among ties, the axes the cases reach, and the refusals of yfv2_ncnn_post and of the Python wrappers, which come
before anything is launched (so no GPU is needed)."""
import ctypes
import os

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import ncnn_space as ns
from oracle import ncnn_post as onp

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = {c["name"]: c for c in ns.cases_all() + ns.limit_cases()}


def golden():
    g = np.load(os.path.join(HERE, "golden", "ncnn_space.npz"))
    out = {}
    for name in g["names"]:
        name = str(name)
        A, C, W, H, sw, sh = [int(v) for v in g[name + "_params"]]
        thr, nms = g[name + "_fparams"]
        c = dict(CASES[name])
        c.update(out2=g[name + "_out2"], out3=g[name + "_out3"], A=A, C=C, W=W, H=H, src=(sw, sh), thresh=thr, nms=nms,
                 anchors=g[name + "_anchors"], boxes=g[name + "_boxes"], scores=g[name + "_scores"], cates=g[name + "_cates"])
        out[name] = c
    return out


GOLDEN = golden()


def run_oracle(c):
    sw, sh = ns.scales(c)
    return onp.ncnn_post(c["out2"], c["out3"], c["A"], c["C"], c["W"], c["H"], c["anchors"], f32(c["thresh"]), f32(c["nms"]),
                         f32(sw), f32(sh))


f32 = np.float32


@pytest.mark.parametrize("name", sorted(GOLDEN))
def test_oracle_matches_the_reference_cpp(name):
    c = GOLDEN[name]
    b, s, k = run_oracle(c)
    assert len(s) == len(c["scores"]), (len(s), len(c["scores"]))
    assert np.array_equal(b, c["boxes"]) and np.array_equal(k, c["cates"])
    assert np.array_equal(s.view(np.uint32), c["scores"].view(np.uint32))


def test_every_case_sits_on_its_side():
    """The claims of every builder hold on the inputs the goldens store (and on the builders' own inputs for the others)."""
    assert set(GOLDEN) | {"geo_a4_640x352"} == set(CASES)
    for name, c in CASES.items():
        ns.check(GOLDEN.get(name, c))
        assert ns.golden_ok(c) == (name in GOLDEN), name


def test_ties_keep_push_order():
    """Cases with equal scores among at most 16 candidates: the reference's rows of one score come in push order."""
    tied = [n for n, c in GOLDEN.items() if ns.push_order_ties(c) > 1]
    assert {"thr_minus2", "thr_minus2_spread", "all_nonpositive", "obj_zero"} <= set(tied)
    for name in tied:
        c = GOLDEN[name]
        cand = ns.candidates(c)
        used = np.zeros(len(cand["score"]), bool)
        order = []
        for box, s, k in zip(c["boxes"], c["scores"], c["cates"]):
            hit = np.flatnonzero(cand["passed"] & ~used & (cand["cate"] == k) & (cand["score"].view(np.uint32) == s.view(np.uint32))
                                 & (cand["box"] == box).all(1))
            assert len(hit), (name, box, s, k)
            used[hit[0]] = True
            order.append(hit[0])
        for i in range(1, len(order)):
            if c["scores"][i] == c["scores"][i - 1]:
                assert order[i] > order[i - 1], (name, i)


def test_cases_reach_every_axis():
    cs = list(CASES.values())
    assert {c["A"] for c in cs} >= {1, 2, 3, 4, 8}
    assert {c["C"] for c in cs} >= {1, 2, 31, 32, 33, 80, 150, 1000, ns.MAX_C}
    assert {(c["H"], c["W"]) for c in cs} >= {(32, 32), (64, 160), (640, 352), (352, 352)}
    lanes = CASES["lane_ties"]["claims"]["cates"]
    pairs = set()
    for slot, k in lanes.items():
        row = CASES["lane_ties"]["out2"].reshape(-1, CASES["lane_ties"]["out2"].shape[-1])[slot // 3, 15:]
        pairs |= {j - k for j in np.flatnonzero(row == row[k]) if j > k}
    assert {32, 64} <= pairs
    thr = {n: CASES[n]["thresh"] for n in ("thr_at_score", "thr_below_score", "thr_minus2", "thr_one", "thr_zero")}
    assert thr["thr_minus2"] == -2 and thr["thr_one"] == 1 and thr["thr_zero"] == 0
    sc = ns.candidates(CASES["thr_at_score"])["score"]
    assert thr["thr_at_score"] in sc and np.nextafter(thr["thr_below_score"], f32(1)) in sc
    assert {float(CASES["touch_nms%g" % v]["nms"]) for v in (0.0, 1.0, -0.1)} == {0.0, 1.0, float(f32(-0.1))}
    counts = {c["claims"]["count"] for c in cs if "count" in c["claims"]}
    assert {1, 63, 64, 65, 128, 129} <= counts
    assert [ns.max_out_edges(5)] == [[1, 4, 5, 6]]
    for A in (1, 3, 8):
        last, first = ns.largest_square(A)
        assert ("limit_a%d_%d" % (A, last)) in CASES and not ns.fits(A, first, first)
    assert ns.largest_square(3) == (672, 704) and ns.largest_square(1) == (1184, 1216) and ns.largest_square(8) == (416, 448)
    for n in ("nonfinite_box", "huge_box", "src_out_of_range", "nan_scores", "chain", "zero_area_identical", "trunc_negative"):
        assert n in CASES


def test_corner_rule():
    """yfv2_ncnn_corner: truncation toward zero; NaN or a truncated value outside the int range gives INT_MIN, as the sample's
    `int = double` compiles to on x86-64 (cvttsd2si)."""
    v = [-0.7, 0.7, -1.5, 2147483647.9, 2147483648.0, -2147483648.9, -2147483649.0, np.nan, np.inf, -np.inf, 3e9, -3e9]
    want = [0, 0, -1, 2147483647, ns.INT_MIN, ns.INT_MIN, ns.INT_MIN, ns.INT_MIN, ns.INT_MIN, ns.INT_MIN, ns.INT_MIN, ns.INT_MIN]
    assert ns.corner(v).tolist() == want


def test_ncnn_post_refusals_come_before_any_launch():
    import yfv2_engine
    lib = yfv2_engine.lib()
    fake = ctypes.c_void_p(256)                               # never dereferenced: every call below fails its host-side check
    anchors = (ctypes.c_float * 32)(*range(1, 33))

    def call(H, W, A, C, max_out, N=1):
        return lib.yfv2_ncnn_post(fake, fake, N, H, W, A, C, anchors, ctypes.c_float(0.3), ctypes.c_float(0.25), ctypes.c_float(1),
                                  ctypes.c_float(1), max_out, fake, fake, fake, fake, None)
    for args in ((352, 352, 0, 80, 10), (352, 352, 9, 80, 10), (352, 352, 3, 0, 10), (352, 352, 3, 32768, 10), (336, 352, 3, 80, 10),
                 (352, 100, 3, 80, 10), (352, 352, 3, 80, 0), (352, 352, 3, 80, -1), (352, 352, 3, 80, 10, 0)):
        assert call(*args) == -1, args
        assert b"bad arguments" in lib.yfv2_last_error()
    for A in (1, 2, 3, 4, 8):
        _, first = ns.largest_square(A)
        assert call(first, first, A, 1, 10) == -3, A
        msg = lib.yfv2_last_error().decode()
        assert "shared memory" in msg and ("%d candidates" % ns.slots(A, first, first)) in msg and str(ns.smem_bytes(ns.slots(A, first, first))) in msg
    assert call(1216, 1184, 1, 1, 10) == -3                   # M = 7030 at a non-square input


class _NoLib:
    def __getattr__(self, name):
        raise AssertionError("the library was called (%s) with tensors that do not fit together" % name)


@pytest.fixture
def shape_checks_only(monkeypatch):
    """CPU tensors stand in for device tensors and any library call fails the test: what remains is the host-side geometry check
    of the wrappers, which must refuse a mismatch before anything is launched."""
    import yfv2_engine
    monkeypatch.setattr(yfv2_engine, "_require_cuda", lambda t, name: None)
    monkeypatch.setattr(yfv2_engine, "lib", lambda: _NoLib())
    return yfv2_engine


def _preds(N=2, A=3, C=80, h=4, w=6):
    return [torch.zeros(N, 4 * A, h, w), torch.zeros(N, A, h, w), torch.zeros(N, C, h, w), torch.zeros(N, 4 * A, h // 2, w // 2),
            torch.zeros(N, A, h // 2, w // 2), torch.zeros(N, C, h // 2, w // 2)]


def mismatched_preds():
    """(label, six tensors) that disagree with preds[0..2] in one place each."""
    out = []
    for i in range(6):
        for dim, delta in ((0, -1), (1, 1), (2, -1), (3, 1)):
            p = _preds()
            shape = list(p[i].shape)
            shape[dim] += delta
            p[i] = torch.zeros(shape)
            out.append(("preds[%d] dim %d %+d" % (i, dim, delta), p))
    p = _preds(h=5, w=6)
    out.append(("odd rows", p))
    out.append(("five tensors", _preds()[:5]))
    return out


@pytest.mark.parametrize("label,preds", mismatched_preds(), ids=[m[0] for m in mismatched_preds()])
def test_head_wrappers_refuse_mismatched_preds(shape_checks_only, label, preds):
    eng = shape_checks_only
    cfg = {"height": preds[0].shape[2] * 16, "width": preds[0].shape[3] * 16, "anchors": [1.0] * 4 * preds[1].shape[1]}
    for fn in (lambda: eng.export_heads(preds), lambda: eng.decode(preds, cfg), lambda: eng.decode_nms(preds, cfg)):
        with pytest.raises(eng.Yfv2Error) as e:
            fn()
        assert "preds" in str(e.value)


def mismatched_outs():
    o2 = (2, 4, 6, 95)
    out = []
    for dim in range(4):
        s = [2, 2, 3, 95]
        s[dim] -= 1
        out.append(("out3 dim %d smaller" % dim, o2, tuple(s)))
        s = [2, 2, 3, 95]
        s[dim] += 1
        out.append(("out3 dim %d larger" % dim, o2, tuple(s)))
    out.append(("out2 odd rows", (2, 5, 6, 95), (2, 2, 3, 95)))
    out.append(("out2 three dims", (4, 6, 95), (2, 3, 95)))
    return out


@pytest.mark.parametrize("label,s2,s3", mismatched_outs(), ids=[m[0] for m in mismatched_outs()])
def test_ncnn_post_refuses_mismatched_out3(shape_checks_only, label, s2, s3):
    eng = shape_checks_only
    with pytest.raises(eng.Yfv2Error) as e:
        eng.ncnn_post(torch.zeros(s2), torch.zeros(s3), 3)
    assert ("out3" in str(e.value) or "out2" in str(e.value)) and "expected" in str(e.value)


def test_ncnn_post_refuses_max_out_below_one(shape_checks_only):
    eng = shape_checks_only
    for m in (0, -3):
        with pytest.raises(eng.Yfv2Error):
            eng.ncnn_post(torch.zeros(1, 2, 2, 95), torch.zeros(1, 1, 1, 95), 3, max_out=m)

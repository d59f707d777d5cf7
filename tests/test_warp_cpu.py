"""Warped views, CPU side: the numpy restatement (tests/warp_oracle.py over the remap, layout, YUV and Bayer oracles and
oracle/resize.py) against outputs of the real cv2.warpAffine / cv2.warpPerspective + crop + cv2.resize
(tests/golden/warp_cases.npz), the library's host inversion against cv2.invert's frozen bits, the descriptor checks of
yfv2_resize_warp_u8 and yfv2_warp_u8 before any launch, and the refusals, windows and sizes of the Python entries."""
import hashlib
import os

import numpy as np
import pytest

import yfv2  # noqa: F401
import remap_oracle as ro
import warp_cases as wc
import warp_oracle as wo
import yfv2_engine as eng


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "warp_cases.npz"))


@pytest.mark.parametrize("c", wc.CASES, ids=[c["name"] for c in wc.CASES])
def test_oracle_matches_cv2(golden, c):
    name = c["name"]
    frame = wc.case_frame(c)
    assert np.array_equal(sha(frame), golden[name + "_in_sha256"]), "the seeded input generator changed"
    M = wc.case_matrix(c, golden)
    img = ro.inner_bgr(frame, c["layout"], c["inner"])
    window = wc.view_window(c)
    warp = wo.warp_window(img, M, c["dsize"], window, c["inverse"])
    if name + "_warp" in golden:
        assert np.array_equal(warp, golden[name + "_warp"])
    assert np.array_equal(sha(warp), golden[name + "_warp_sha256"])
    W, H = c["target"]
    got = wo.resize_planar(img, M, c["dsize"], window, W, H, c["inverse"]).transpose(1, 2, 0)
    if name + "_out" in golden:
        assert np.array_equal(got, golden[name + "_out"])
    assert np.array_equal(sha(got), golden[name + "_sha256"])


def test_cases_cover_the_space(golden):
    assert set(wc.LAYOUTS) == set(eng.LAYOUTS + eng.BAYER_LAYOUTS) and len(wc.LAYOUTS) == 21
    shapes = {(c["M"].shape, c["inverse"]) for c in wc.CASES}
    assert shapes == {((2, 3), False), ((2, 3), True), ((3, 3), False), ((3, 3), True)}
    assert {c["rotate"] for c in wc.CASES} >= {"ROTATE_90_COUNTERCLOCKWISE", "ROTATE_180", "ROTATE_90_CLOCKWISE"}
    assert any(c["size"] == (1, 1) for c in wc.CASES) and any(tuple(c["dsize"]) == (1, 1) for c in wc.CASES)
    assert any(c["view"] for c in wc.CASES) and any(c["inner"] for c in wc.CASES)
    assert any(c["size"] == (1080, 1920) for c in wc.CASES)
    assert wc.FROM_GOLDEN == {k[:-2] for k in golden.files if k.endswith("_M")}
    # the horizon cases have a row where W is exactly 0, and the birdseye ones a horizon inside the output
    for name, row in (("bgr_horizon_row", 64), ("bayer_gb_horizon_row", 64)):
        c = [c for c in wc.CASES if c["name"] == name][0]
        m = wo.dst_to_src(c["M"], c["inverse"])[1]
        assert m[7] * row + m[8] == 0 and m[6] == 0
        xy, code = wo.warp_maps(m, True, 0, row, c["dsize"][0], 1)
        assert (xy == 0).all() and (code == 0).all()
    c = [c for c in wc.CASES if c["name"] == "bgr_birdseye"][0]
    m = wo.dst_to_src(wc.case_matrix(c, golden), True)[1]
    w0 = [m[7] * y + m[8] for y in (0, c["dsize"][1] - 1)]
    assert w0[0] < 0 < w0[1]


def test_ties_reach_half_way_roundings():
    """The tie cases put half-way values into cvRound: rounding half away from zero would change their coordinates."""
    for name in ("bgr_affine_ties", "bgr_persp_affine_row_ties", "gray_persp_ties"):
        c = [c for c in wc.CASES if c["name"] == name][0]
        persp, m = wo.dst_to_src(c["M"], c["inverse"])
        dw, dh = c["dsize"]
        x = np.arange(dw, dtype=np.float64)[None, :]
        y = np.arange(dh, dtype=np.float64)[:, None]
        if persp:
            W = 32.0 / ((m[7] * y + m[8]) + m[6] * x)
            vals = [((m[1] * y + m[2]) + m[0] * x) * W, ((m[4] * y + m[5]) + m[3] * x) * W]
        else:
            vals = [(m[0] * x) * 1024.0, (m[1] * y + m[2]) * 1024.0]
        assert any((np.abs(v - np.floor(v)) == 0.5).any() for v in vals), name


def test_affine_bound_cases_sit_just_inside():
    for name in ("bgr_affine_bound_row", "bgr_affine_bound_x"):
        c = [c for c in wc.CASES if c["name"] == name][0]
        persp, m = wo.dst_to_src(c["M"], c["inverse"])
        assert wo.affine_fits(m, *c["dsize"])
        big = m.copy()
        big[2 if name.endswith("row") else 0] *= 1.0 + 2.0 ** -9
        assert not wo.affine_fits(big, *c["dsize"])


def test_host_inversion_equals_cv2_invert(golden):
    """yfv2_warp_matrix's perspective inversion against cv2.invert(M, DECOMP_LU)'s frozen results on 3000 random,
    ill-conditioned, singular and camera-like matrices: every bit, and the singular ones refused."""
    mats = wc.inv_matrices()
    oks = golden["inv_ok"]
    got = np.zeros((len(mats), 3, 3), np.float64)
    refused = 0
    for k, m in enumerate(mats):
        if not oks[k]:
            with pytest.raises(eng.Yfv2Error, match="warp_matrix: singular matrix"):
                eng.warp_matrix(m)
            refused += 1
            continue
        got[k] = eng.warp_matrix(m)
    assert refused == int((~oks).sum()) > 0
    assert np.array_equal(got[:64], golden["inv_head"])
    assert np.array_equal(sha(got), golden["inv_sha256"])


def test_host_affine_inversion_is_the_oracles(golden):
    """The affine inverse is pinned through bytes (make_golden_warp.py: warpAffine(M) equals warpAffine(inv(M),
    WARP_INVERSE_MAP) with the oracle's inverse); the library's equals the oracle's bit for bit, and inverse=True passes M as is."""
    rs = np.random.RandomState(5)
    mats = [wc.case_matrix(c, golden) for c in wc.CASES if c["M"].shape == (2, 3) and not c["inverse"]]
    mats += [rs.uniform(-3, 3, (2, 3)) * 10.0 ** rs.randint(-3, 3) for _ in range(500)]
    for M in mats:
        want = wo.invert_affine(M)
        want = np.append(want, [0.0, 0.0, 1.0]).reshape(3, 3)
        assert np.array_equal(eng.warp_matrix(M), want), M
        assert np.array_equal(eng.warp_matrix(M, inverse=True)[:2], M)
        assert np.array_equal(eng.warp_matrix(M, inverse=True)[2], [0, 0, 1])


FAKE = 0x1000                                                  # never dereferenced: every check runs on the host first


def warp_frames_c(*descs):
    arr = (eng.WarpFrame * len(descs))()
    for a, d in zip(arr, descs):
        a.kind, a.x0, a.y0, a.w, a.h = d["kind"], d["x0"], d["y0"], d["w"], d["h"]
        b = a.f.bgr
        b.data, b.w, b.h, b.pitch = d["data"], d["fw"], d["fh"], d["pitch"]
        a.m[:] = list(d["m"]) + [0.0] * (9 - len(d["m"]))
        a.perspective, a.inverse, a.dw, a.dh = d["perspective"], d["inverse"], d["dw"], d["dh"]
    return arr


GOOD = dict(kind=eng.JPEG_SRC_BGR, x0=3, y0=5, w=600, h=400, data=FAKE, fw=640, fh=480, pitch=1920,
            m=(0.9, 0.1, 5.0, -0.1, 0.9, 7.0), perspective=0, inverse=0, dw=640, dh=480)
PERSP = dict(GOOD, m=(1.0, 0.1, 5.0, 0.0, 1.2, 7.0, 1e-4, 2e-4, 1.0), perspective=1)


def test_warp_abi_rejects_bad_descriptors_before_any_launch():
    """Each bad field refused by both entries with its reason, naming the entry and the frame; one in a later launch's chunk too."""
    nan, inf = float("nan"), float("inf")
    faults = [(dict(kind=eng.JPEG_SRC_GRAY), "kind must be"), (dict(kind=6), "kind must be"), (dict(data=None), "null data"),
              (dict(pitch=1919), "pitch < 3 * w"),
              (dict(perspective=2), "perspective must be 0 or 1"), (dict(inverse=-1), "inverse must be 0 or 1"),
              (dict(dw=0), "dw and dh must be in 1..32767"), (dict(dh=32768), "dw and dh must be in 1..32767"),
              (dict(m=(0.9, 0.1, nan, -0.1, 0.9, 7.0)), "matrix entries must be finite"),
              (dict(m=(0.9, 0.1, 5.0, -0.1, inf, 7.0), inverse=1), "matrix entries must be finite"),
              (dict(m=(1.0, 2.0, 5.0, 2.0, 4.0, 7.0)), "singular matrix"),
              (dict(m=(0.0,) * 6), "singular matrix"),
              (dict(PERSP, m=(1, 2, 3, 2, 4, 6, 0, 0, 1)), "singular matrix"),
              (dict(PERSP, m=(1, 0, 0, 0, 1, 0, 0, 0, nan)), "matrix entries must be finite"),
              (dict(PERSP, m=(1e-103, 0, 0, 0, 1e-103, 0, 0, 0, 1e-103)), "the inverse has non-finite entries"),
              (dict(m=(1e-160, 0, 0, 0, 1e-160, 0)), "the inverse has non-finite entries"),
              (dict(m=(1.0, 0.0, 1048576.0, 0.0, 1.0, 0.0), inverse=1), "affine coordinates reach 2^30"),
              (dict(m=(1.0, 0.0, 0.0, 0.0, 1.0, -1048576.0), inverse=1), "affine coordinates reach 2^30"),
              (dict(m=(1.0, 0.0, 0.0, 0.0, 1024.0, 0.0), inverse=1, dw=32767, dh=1025, w=5, h=5), "affine coordinates"),
              (dict(m=(1677.0, 0.0, 0.0, 0.0, 1.0, 0.0), inverse=1), "affine coordinates"),
              (dict(m=(1.0, 0.0, 0.0, -1677.0, 1.0, 0.0), inverse=1), "affine coordinates"),
              (dict(w=0), "window empty or outside the output"), (dict(h=-1), "window"), (dict(x0=-1), "window"),
              (dict(y0=-1), "window"), (dict(x0=41), "window"), (dict(y0=81), "window"), (dict(x0=1 << 30, w=1 << 30), "window")]
    L = eng.lib()
    dst = eng.ctypes.c_void_p(FAKE)
    dsts = (eng.ctypes.c_void_p * 200)(*([FAKE] * 200))
    for n in (0, -1):
        assert L.yfv2_resize_warp_u8(warp_frames_c(GOOD), n, 352, 352, dst, None) == -1
        assert b"resize_warp_u8: null frames / dst or N <= 0" in L.yfv2_last_error()
        assert L.yfv2_warp_u8(warp_frames_c(GOOD), n, dsts, None) == -1
        assert b"warp_u8: null frames / dst or N <= 0" in L.yfv2_last_error()
    assert L.yfv2_resize_warp_u8(warp_frames_c(GOOD), 1, 352, 352, None, None) == -1
    assert L.yfv2_warp_u8(warp_frames_c(GOOD), 1, None, None) == -1
    for H, W in ((0, 352), (352, 0), (32769, 352), (352, 32769)):
        assert L.yfv2_resize_warp_u8(warp_frames_c(GOOD), 1, H, W, dst, None) == -1
        assert b"resize_warp_u8: target" in L.yfv2_last_error()
    for f, why in faults:
        bad = dict(GOOD, **f)
        assert L.yfv2_resize_warp_u8(warp_frames_c(GOOD, bad), 2, 352, 352, dst, None) == -1, f
        err = L.yfv2_last_error()
        assert b"resize_warp_u8: frame 1: " + why.encode() in err, (f, err)
        assert L.yfv2_warp_u8(warp_frames_c(PERSP, bad), 2, dsts, None) == -1, f
        assert b"warp_u8: frame 1: " + why.encode() in L.yfv2_last_error(), f
    nulls = (eng.ctypes.c_void_p * 2)(FAKE, None)
    assert L.yfv2_warp_u8(warp_frames_c(GOOD, PERSP), 2, nulls, None) == -1
    assert b"warp_u8: frame 1: null dst" in L.yfv2_last_error()
    many = warp_frames_c(*([GOOD] * 130 + [dict(GOOD, data=None)]))
    assert L.yfv2_resize_warp_u8(many, 131, 352, 352, dst, None) == -1
    assert b"frame 130: null data" in L.yfv2_last_error()
    # just inside the affine bound is accepted by the host checks (the matrix query runs them without a launch)
    out = (eng.ctypes.c_double * 9)()
    ok = warp_frames_c(dict(GOOD, m=(1.0, 0.0, 1048575.0, 0.0, 1.0, 0.0), inverse=1, x0=0, y0=0, w=8, h=8, dw=8, dh=8))
    assert L.yfv2_warp_matrix(ok, out) == 0 and list(out) == [1, 0, 1048575, 0, 1, 0, 0, 0, 1]


def test_descriptor_layout_and_encoder_union_unchanged():
    """The warp descriptor holds the encoder's frame union, which keeps its size, then the matrix and its four ints."""
    assert eng.ctypes.sizeof(eng._EncFrame) == 56
    assert eng.WarpFrame.f.offset == 24 and eng.WarpFrame.m.offset == 80
    assert eng.WarpFrame.perspective.offset == 152 and eng.WarpFrame.dh.offset == 164 and eng.ctypes.sizeof(eng.WarpFrame) == 168
    assert eng.ctypes.sizeof(eng.RemapFrame) == 24 + 56 + 40
    assert eng.lib().yfv2_abi_version() == 1


def test_warp_view_copies_its_matrix_and_refuses_bad_shapes():
    M = np.array([[1.0, 0.0, 2.0], [0.0, 1.0, 3.0]])
    v = eng.WarpView(np.zeros((4, 4, 3), np.uint8), M, (10, 8))
    M[0, 2] = 99.0
    assert v.m == (1.0, 0.0, 2.0, 0.0, 1.0, 3.0) and not v.perspective and (v.dw, v.dh, v.w, v.h) == (10, 8, 10, 8)
    v = eng.WarpView(np.zeros((4, 4, 3), np.uint8), [[1, 0, 0], [0, 1, 0], [0, 0, 1]], (10, 8), 2, 3, inverse=True)
    assert v.perspective and v.inverse and (v.x0, v.y0, v.w, v.h) == (2, 3, 8, 5) and all(type(a) is float for a in v.m)
    for bad, msg in (([[1, 0], [0, 1]], "2x3 .* or 3x3"), (np.zeros((3, 4)), "2x3"), ([1, 2, 3, 4, 5, 6], "2x3"),
                     ("abc", "matrix of numbers|2x3")):
        with pytest.raises(eng.Yfv2Error, match="WarpView: M must be " + msg):
            eng.WarpView(np.zeros((4, 4, 3), np.uint8), bad, (10, 8))
    with pytest.raises(eng.Yfv2Error, match="dsize must be"):
        eng.WarpView(np.zeros((4, 4, 3), np.uint8), M, (10, 8, 3))


def test_python_entries_refuse_bad_views_before_anything_runs():
    bgr = np.zeros((30, 40, 3), np.uint8)
    A = [[0.9, 0.1, 2.0], [-0.1, 0.9, 3.0]]
    maps = object.__new__(eng.RemapMaps)
    maps.xy, maps.code, maps.mw, maps.mh = None, None, 64, 48
    cases = [
        ([eng.WarpView(bgr, A, (64, 48), 0, 0, 65, 48)], "bgr", "not inside the 64x48 output"),
        ([eng.WarpView(bgr, A, (64, 48), -1, 0, 5, 5)], "bgr", "not inside"),
        ([eng.WarpView(bgr, A, (64, 48), 5, 5, 0, 3)], "bgr", "not inside"),
        ([eng.WarpView(bgr, A, (0, 48))], "bgr", "dsize 0x48 outside 1..32767"),
        ([eng.WarpView(bgr, A, (40000, 48), 0, 0, 5, 5)], "bgr", "dsize 40000x48"),
        ([eng.WarpView(bgr, [[1, 2, 0], [2, 4, 0]], (64, 48))], "bgr", "frame 0 \\(bgr view\\): singular matrix"),
        ([eng.WarpView(bgr, [[1e-103, 0, 0], [0, 1e-103, 0], [0, 0, 1e-103]], (64, 48))], "bgr", "non-finite"),
        ([eng.WarpView(bgr, [[1, 0, 2e6], [0, 1, 0]], (64, 48), inverse=True)], "bgr", "affine coordinates reach 2\\^30"),
        ([eng.WarpView(bgr, [[1, 0, float("nan")], [0, 1, 0]], (64, 48))], "bgr", "matrix entries must be finite"),
        ([eng.WarpView(bgr, A, (64, 48))], "nv12", "frame 0"), ([eng.WarpView(bgr.astype(np.int8), A, (64, 48))], "bgr", "uint8"),
        ([eng.WarpView(eng.WarpView(bgr, A, (64, 48)), A, (64, 48))], "bgr", "a WarpView of a WarpView"),
        ([eng.WarpView(eng.RemapView(bgr, maps), A, (64, 48))], "bgr", "a WarpView of a RemapView"),
        ([eng.RemapView(eng.WarpView(bgr, A, (64, 48)), maps)], "bgr", "a RemapView of a WarpView"),
        ([bgr, eng.WarpView(bgr, A, (64, 48)), eng.WarpView(np.zeros((31, 40), np.uint8), A, (64, 48))], ["bgr", "bgr", "nv12"],
         "frame 2"),
    ]
    entries = {"resize_frames": lambda frames, layout: eng.resize_frames(frames, 352, 352, layout, device="cuda:0"),
               "warp_frames": lambda frames, layout: eng.warp_frames(frames, layout, device="cuda:0"),
               "encode_jpeg": lambda frames, layout: eng.encode_jpeg(frames, layout=layout, device="cuda:0")}
    for frames, layout, msg in cases:
        for name, call in entries.items():
            with pytest.raises(eng.Yfv2Error, match=msg) as e:
                call(frames, layout)
            assert str(e.value).startswith(name + ": "), (layout, str(e.value))
    with pytest.raises(eng.Yfv2Error, match="warp_frames: frame 1 is a ndarray, not a WarpView"):
        eng.warp_frames([eng.WarpView(bgr, A, (64, 48)), bgr], "bgr", device="cuda:0")
    with pytest.raises(eng.Yfv2Error, match="remap_frames: frame 0 is a WarpView, not a RemapView"):
        eng.remap_frames([eng.WarpView(bgr, A, (64, 48))], "bgr", device="cuda:0")
    with pytest.raises(eng.Yfv2Error, match="encode_jpeg: output 1: region .* is not inside the 64x48 view"):
        eng.encode_jpeg([bgr, eng.WarpView(bgr, A, (64, 48))], layout="bgr", regions=[(0, 0, 0, 4, 4), (1, 60, 0, 5, 4)],
                        device="cuda:0")


def test_crop_frame_windows_of_views_compose_and_stay_inside():
    nv12 = np.zeros((72, 80), np.uint8)
    H = [[1, 0.1, 0], [0, 1, 0], [0, 1e-3, 1]]
    v = eng.WarpView(nv12, H, (64, 48))
    assert (v.x0, v.y0, v.w, v.h) == (0, 0, 64, 48) and eng.frame_size(v, "nv12") == (48, 64)
    w1 = eng.crop_frame(v, "nv12", 5, 7, 41, 31)                 # odd offsets and sizes: a window of the warped image
    assert isinstance(w1, eng.WarpView) and (w1.x0, w1.y0, w1.w, w1.h) == (5, 7, 41, 31)
    assert w1.m == v.m and w1.perspective and (w1.dw, w1.dh) == (64, 48)
    w2 = eng.crop_frame(w1, "nv12", 3, 1, 37, 29)
    assert (w2.x0, w2.y0, w2.w, w2.h) == (8, 8, 37, 29) and eng.frame_size(w2, "nv12") == (29, 37)
    for x0, y0, w, h in [(0, 0, 38, 29), (0, 0, 37, 30), (1, 0, 37, 29), (0, -1, 5, 5), (0, 0, 0, 1)]:
        with pytest.raises(eng.Yfv2Error, match="crop_frame: window .* is not inside the 37x29 frame"):
            eng.crop_frame(w2, "nv12", x0, y0, w, h)
    assert eng.WarpView(nv12, H, (64, 48), 10, 20).w == 54 and eng.WarpView(nv12, H, (64, 48), 10, 20).h == 28
    inv = eng.crop_frame(eng.WarpView(nv12, H, (64, 48), inverse=True), "nv12", 1, 2, 3, 4)
    assert inv.inverse

"""Lens-corrected views, CPU side: the numpy restatement (tests/remap_oracle.py over the layout, YUV and Bayer oracles and
oracle/resize.py) and the library's map conversion against outputs of the real cv2.convertMaps + cv2.remap + crop + cv2.resize
(tests/golden/remap_cases.npz), the descriptor checks of yfv2_resize_remap_u8 and yfv2_remap_u8 before any launch, and the
refusals, windows and sizes of the Python entries."""
import hashlib
import os

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import remap_cases as rc
import remap_oracle as ro
import yfv2_engine as eng


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def maps_sha(m1, m2):
    return sha(np.concatenate([np.ascontiguousarray(m1).reshape(-1).view(np.uint8),
                               np.ascontiguousarray(m2).reshape(-1).view(np.uint8)]))


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "remap_cases.npz"))


@pytest.mark.parametrize("c", rc.CASES, ids=[c["name"] for c in rc.CASES])
def test_oracle_matches_cv2(golden, c):
    name = c["name"]
    frame = rc.case_frame(c)
    assert np.array_equal(sha(frame), golden[name + "_in_sha256"]), "the seeded input generator changed"
    m1, m2 = rc.fixed_maps(c, golden)
    assert np.array_equal(maps_sha(m1, m2), golden[name + "_maps_sha256"]), "maps or their conversion differ from cv2's"
    img = ro.inner_bgr(frame, c["layout"], c["inner"])
    window = rc.view_window(c)
    rem = ro.remap_window(img, m1, m2, window)
    if name + "_remap" in golden:
        assert np.array_equal(rem, golden[name + "_remap"])
    assert np.array_equal(sha(rem), golden[name + "_remap_sha256"])
    W, H = c["target"]
    got = ro.resize_planar(img, m1, m2, window, W, H).transpose(1, 2, 0)
    if name + "_out" in golden:
        assert np.array_equal(got, golden[name + "_out"])
    assert np.array_equal(sha(got), golden[name + "_sha256"])


@pytest.mark.parametrize("c", [c for c in rc.CASES if c["form"] in ("float2", "c2")],
                         ids=[c["name"] for c in rc.CASES if c["form"] in ("float2", "c2")])
def test_library_map_conversion_equals_cv2(golden, c):
    """RemapMaps' conversion (eng.convert_maps, torch on the CPU here) of the case's float maps gives cv2.convertMaps' maps."""
    m1, m2 = rc.case_maps(c)
    mx, my = (m1[..., 0], m1[..., 1]) if m2 is None else (m1, m2)
    xy, code = eng.convert_maps(torch.from_numpy(np.ascontiguousarray(mx)), torch.from_numpy(np.ascontiguousarray(my)))
    assert xy.dtype == torch.int16 and code.dtype == torch.int16
    assert np.array_equal(maps_sha(xy.numpy(), code.numpy()), golden[c["name"] + "_maps_sha256"])


def test_convert_maps_edge_values(golden):
    """NaN, +-inf and huge values, saturation and half-way ties, against cv2.convertMaps and the values cv2 4.13 gives."""
    e1, e2 = golden["edge_map1"][0], golden["edge_map2"][0]
    o1, o2 = ro.convert_maps(rc.EDGE_VALUES, np.zeros_like(rc.EDGE_VALUES))
    assert np.array_equal(o1, e1) and np.array_equal(o2, e2)
    xy, code = eng.convert_maps(torch.from_numpy(rc.EDGE_VALUES), torch.zeros(len(rc.EDGE_VALUES)))
    assert np.array_equal(xy.numpy(), e1) and np.array_equal(code.numpy().view(np.uint16), e2)
    pinned = {0: (-32768, 0), 1: (-32768, 0), 2: (-32768, 0), 3: (-32768, 0), 4: (-32768, 0), 5: (32767, 0), 7: (32767, 28),
              8: (0, 2), 9: (0, 4), 10: (0, 0)}
    for k, (x0, code) in pinned.items():
        assert (int(e1[k, 0]), int(e2[k])) == (x0, code), rc.EDGE_VALUES[k]


def test_weight_table_is_the_closed_form_the_kernel_uses():
    """cv2's table, computed cv2's way, is 32 (32 - i)(32 - j), 32 (32 - i) j, 32 i (32 - j), 32 i j: no sum correction fires."""
    i, j = np.meshgrid(np.arange(32), np.arange(32), indexing="ij")
    closed = 32 * np.stack([(32 - i) * (32 - j), (32 - i) * j, i * (32 - j), i * j], -1).reshape(1024, 4)
    assert np.array_equal(ro.weight_table(), closed) and (closed.sum(1) == 32768).all()


def test_cases_cover_every_layout_and_map_form():
    assert set(rc.LAYOUTS) == set(eng.LAYOUTS + eng.BAYER_LAYOUTS) and len(rc.LAYOUTS) == 21
    assert {c["form"] for c in rc.CASES} == {"float2", "c2", "convert", "fixed"}
    assert {c["map"][0] for c in rc.CASES} == {"undistort", "fisheye", "random", "grid64", "junk", "cv2fixed"}
    assert any(c["size"] == (1, 1) for c in rc.CASES) and any(c["view"] for c in rc.CASES)
    assert any(c["map"][1] < c["size"][1] for c in rc.CASES) and any(c["map"][1] > c["size"][1] for c in rc.CASES)
    grid = [c for c in rc.CASES if c["map"][0] == "grid64"][0]
    m1, m2 = rc.fixed_maps(grid)
    assert len(np.unique(m2)) == 1024


FAKE = 0x1000                                                  # never dereferenced: every check runs on the host first


def remap_frames_c(*descs):
    arr = (eng.RemapFrame * len(descs))()
    for a, d in zip(arr, descs):
        a.kind, a.x0, a.y0, a.w, a.h = d["kind"], d["x0"], d["y0"], d["w"], d["h"]
        b = a.f.bgr
        b.data, b.w, b.h, b.pitch = d["data"], d["fw"], d["fh"], d["pitch"]
        m = a.map
        m.xy, m.xy_pitch, m.code, m.code_pitch, m.mw, m.mh = d["xy"], d["xy_pitch"], d["code"], d["code_pitch"], d["mw"], d["mh"]
    return arr


GOOD = dict(kind=eng.JPEG_SRC_BGR, x0=3, y0=5, w=600, h=400, data=FAKE, fw=640, fh=480, pitch=1920, xy=FAKE, xy_pitch=2560,
            code=FAKE, code_pitch=1280, mw=640, mh=480)


def test_remap_abi_rejects_bad_descriptors_before_any_launch():
    """Each bad field refused by both entries with its reason, naming the entry and the frame; one in a later launch's chunk too."""
    faults = [(dict(kind=eng.JPEG_SRC_GRAY), "kind must be"), (dict(kind=6), "kind must be"), (dict(kind=-1), "kind must be"),
              (dict(data=None), "null data"), (dict(pitch=1919), "pitch < 3 * w"), (dict(fw=0), "w and h must be > 0"),
              (dict(xy=None), "null map plane"), (dict(code=None), "null map plane"),
              (dict(mw=0), "map sides"), (dict(mh=-1), "map sides"), (dict(mw=32768, xy_pitch=4 * 32768, code_pitch=2 * 32768),
                                                                     "map sides"),
              (dict(xy_pitch=2556), "xy must be 4-byte aligned, xy_pitch >= 4 * mw"), (dict(xy_pitch=2562), "xy must be 4-byte aligned"),
              (dict(xy=FAKE + 2), "xy must be 4-byte aligned"), (dict(code_pitch=1278), "code must be 2-byte aligned, code_pitch >= 2 * mw"),
              (dict(code_pitch=1281), "code must be 2-byte aligned"), (dict(code=FAKE + 1), "code must be 2-byte aligned"),
              (dict(w=0), "window empty or outside the map"), (dict(h=-1), "window"), (dict(x0=-1), "window"),
              (dict(y0=-1), "window"), (dict(x0=41), "window"), (dict(y0=81), "window"),
              (dict(x0=1 << 30, w=1 << 30), "window")]
    L = eng.lib()
    dst = eng.ctypes.c_void_p(FAKE)
    dsts = (eng.ctypes.c_void_p * 200)(*([FAKE] * 200))
    for n in (0, -1):
        assert L.yfv2_resize_remap_u8(remap_frames_c(GOOD), n, 352, 352, dst, None) == -1
        assert b"resize_remap_u8: null frames / dst or N <= 0" in L.yfv2_last_error()
        assert L.yfv2_remap_u8(remap_frames_c(GOOD), n, dsts, None) == -1
        assert b"remap_u8: null frames / dst or N <= 0" in L.yfv2_last_error()
    assert L.yfv2_resize_remap_u8(remap_frames_c(GOOD), 1, 352, 352, None, None) == -1
    assert L.yfv2_remap_u8(remap_frames_c(GOOD), 1, None, None) == -1
    for H, W in ((0, 352), (352, 0), (32769, 352), (352, 32769)):
        assert L.yfv2_resize_remap_u8(remap_frames_c(GOOD), 1, H, W, dst, None) == -1
        assert b"resize_remap_u8: target" in L.yfv2_last_error()
    for f, why in faults:
        bad = dict(GOOD, **f)
        assert L.yfv2_resize_remap_u8(remap_frames_c(GOOD, bad), 2, 352, 352, dst, None) == -1, f
        err = L.yfv2_last_error()
        assert b"resize_remap_u8: frame 1: " + why.encode() in err, (f, err)
        assert L.yfv2_remap_u8(remap_frames_c(GOOD, bad), 2, dsts, None) == -1, f
        assert b"remap_u8: frame 1: " + why.encode() in L.yfv2_last_error(), f
    nulls = (eng.ctypes.c_void_p * 2)(FAKE, None)
    assert L.yfv2_remap_u8(remap_frames_c(GOOD, GOOD), 2, nulls, None) == -1
    assert b"remap_u8: frame 1: null dst" in L.yfv2_last_error()
    many = remap_frames_c(*([GOOD] * 130 + [dict(GOOD, data=None)]))
    assert L.yfv2_resize_remap_u8(many, 131, 352, 352, dst, None) == -1
    assert b"frame 130: null data" in L.yfv2_last_error()


def test_descriptor_layout_and_encoder_union_unchanged():
    """The remap descriptor holds the encoder's frame union, which keeps its size; the map is 40 bytes."""
    assert eng.ctypes.sizeof(eng._EncFrame) == eng.ctypes.sizeof(eng.Yuv420Frame)
    assert eng.ctypes.sizeof(eng.RemapMap) == 40
    assert eng.RemapFrame.f.offset == 24 and eng.ctypes.sizeof(eng.RemapFrame) == 24 + 56 + 40
    assert eng.lib().yfv2_abi_version() == 1


def cpu_maps(mw, mh):
    """A RemapMaps whose planes stay on the CPU: enough for the checks that run before anything is placed on a device."""
    m = object.__new__(eng.RemapMaps)
    m.xy, m.code = torch.zeros((mh, mw, 2), dtype=torch.int16), torch.zeros((mh, mw), dtype=torch.int16)
    m.mw, m.mh = mw, mh
    return m


def test_remap_maps_refuse_what_cv2_refuses():
    f = np.zeros((20, 30), np.float32)
    cases = [((f.astype(np.float64), f), "float32, int16 or uint16"), ((f, f.astype(np.float64)), "float32, int16 or uint16"),
             ((f.astype(np.int32), f), "float32, int16 or uint16"), ((f, f[:, :29]), "two float32 \\[h, w\\] planes"),
             ((f, np.zeros((20, 30), np.int16)), "two float32"), ((f, None), "a single float map must be float32 \\[h, w, 2\\]"),
             ((np.zeros((20, 30, 3), np.float32), None), "\\[h, w, 2\\]"), ((np.zeros((20, 30, 2), np.float32), f), "two float32"),
             ((np.zeros((20, 30, 2), np.int16), None), "needs map2 uint16"),
             ((np.zeros((20, 30, 2), np.int16), np.zeros((20, 29), np.uint16)), "needs map2 uint16"),
             ((np.zeros((20, 30), np.int16), np.zeros((20, 30), np.uint16)), "int16 \\[h, w, 2\\]"),
             ((np.zeros((20, 30, 2), np.uint16), np.zeros((20, 30), np.uint16)), "map1 must be float32 or int16"),
             ((np.zeros((0, 30), np.float32), np.zeros((0, 30), np.float32)), "map sides"),
             ((np.zeros((1, 32767), np.float32), np.zeros((1, 32767), np.float32)), "map sides must be in 1..32766"),
             ((torch.zeros((20, 30)), torch.zeros((20, 30), dtype=torch.float64)), "two float32")]
    for (m1, m2), msg in cases:
        with pytest.raises(eng.Yfv2Error, match="RemapMaps: .*" + msg):
            eng.RemapMaps(m1, m2)
    with pytest.raises(eng.Yfv2Error, match="CUDA device"):
        eng.RemapMaps(f, f, device="cpu")
    with pytest.raises(eng.Yfv2Error, match="RemapView: maps must be a RemapMaps"):
        eng.RemapView(np.zeros((4, 4, 3), np.uint8), (f, f))


def test_python_entries_refuse_bad_views_before_anything_runs():
    m = cpu_maps(64, 48)
    bgr = np.zeros((30, 40, 3), np.uint8)
    cases = [
        ([eng.RemapView(bgr, m, 0, 0, 65, 48)], "bgr", "not inside the 64x48 map"),
        ([eng.RemapView(bgr, m, -1, 0, 5, 5)], "bgr", "not inside"), ([eng.RemapView(bgr, m, 60, 40, 5, 5)], "bgr", "not inside"),
        ([eng.RemapView(bgr, m, 5, 5, 0, 3)], "bgr", "not inside"),
        ([eng.RemapView(bgr, m)], "nv12", "frame 0"), ([eng.RemapView(bgr.astype(np.int8), m)], "bgr", "uint8"),
        ([eng.RemapView(eng.RemapView(bgr, m), m)], "bgr", "RemapView of a RemapView"),
        ([eng.RemapView(bgr, m)], "bayer", "layout"),
        ([bgr, eng.RemapView(bgr, m), eng.RemapView(np.zeros((31, 40), np.uint8), m)], ["bgr", "bgr", "nv12"], "frame 2"),
    ]
    entries = {"resize_frames": lambda frames, layout: eng.resize_frames(frames, 352, 352, layout, device="cuda:0"),
               "remap_frames": lambda frames, layout: eng.remap_frames(frames, layout, device="cuda:0"),
               "encode_jpeg": lambda frames, layout: eng.encode_jpeg(frames, layout=layout, device="cuda:0")}
    for frames, layout, msg in cases:
        for name, call in entries.items():
            with pytest.raises(eng.Yfv2Error, match=msg) as e:
                call(frames, layout)
            assert str(e.value).startswith(name + ": "), (layout, str(e.value))
    with pytest.raises(eng.Yfv2Error, match="remap_frames: frame 1 is a ndarray, not a RemapView"):
        eng.remap_frames([eng.RemapView(bgr, m), bgr], "bgr", device="cuda:0")
    with pytest.raises(eng.Yfv2Error, match="encode_jpeg: output 1: region .* is not inside the 64x48 view"):
        eng.encode_jpeg([bgr, eng.RemapView(bgr, m)], layout="bgr", regions=[(0, 0, 0, 4, 4), (1, 60, 0, 5, 4)], device="cuda:0")


def test_crop_frame_windows_of_views_compose_and_stay_inside():
    m = cpu_maps(64, 48)
    nv12 = np.zeros((72, 80), np.uint8)
    v = eng.RemapView(nv12, m)
    assert (v.x0, v.y0, v.w, v.h) == (0, 0, 64, 48) and eng.frame_size(v, "nv12") == (48, 64)
    w1 = eng.crop_frame(v, "nv12", 5, 7, 41, 31)                 # odd offsets and sizes: a window of the remapped image
    assert isinstance(w1, eng.RemapView) and (w1.x0, w1.y0, w1.w, w1.h) == (5, 7, 41, 31) and w1.maps is m
    w2 = eng.crop_frame(w1, "nv12", 3, 1, 37, 29)
    assert (w2.x0, w2.y0, w2.w, w2.h) == (8, 8, 37, 29) and eng.frame_size(w2, "nv12") == (29, 37)
    for x0, y0, w, h in [(0, 0, 38, 29), (0, 0, 37, 30), (1, 0, 37, 29), (0, -1, 5, 5), (0, 0, 0, 1)]:
        with pytest.raises(eng.Yfv2Error, match="crop_frame: window .* is not inside the 37x29 frame"):
            eng.crop_frame(w2, "nv12", x0, y0, w, h)
    assert eng.RemapView(nv12, m, 10, 20).w == 54 and eng.RemapView(nv12, m, 10, 20).h == 28

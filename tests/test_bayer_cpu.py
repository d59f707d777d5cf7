"""Raw Bayer frames, CPU side: the numpy restatement (tests/bayer_oracle.py over oracle/resize.py) against outputs of the real
cv2.cvtColor(COLOR_Bayer??2BGR / _EA) + crop + cv2.resize / cv2.imencode (tests/golden/bayer_cases.npz), the descriptor checks of
yfv2_resize_bayer_u8 and of the JPEG encoder's plan before any launch, and the refusals, windows and sizes of the Python entries."""
import hashlib
import os

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import bayer_cases as bc
import bayer_oracle as bo
import jpeg_encode_cases as jc
import yfv2_engine as eng


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "bayer_cases.npz"))


@pytest.mark.parametrize("case", bc.CASES, ids=[c[0] for c in bc.CASES])
def test_oracle_matches_cv2(golden, case):
    name, layout, _, _, (H, W), _, _ = case
    raw = bc.case_input(case)
    assert np.array_equal(sha(raw), golden[name + "_in_sha256"]), "the seeded input generator changed"
    bgr = bo.window_bgr(raw, layout, *bc.window_of(case))
    if name + "_bgr" in golden:
        assert np.array_equal(bgr, golden[name + "_bgr"])
    assert np.array_equal(sha(bgr), golden[name + "_bgr_sha256"])
    got = bo.resize_planar(raw, layout, W, H, bc.window_of(case)).transpose(1, 2, 0)
    if name + "_out" in golden:
        assert np.array_equal(got, golden[name + "_out"])
    assert np.array_equal(sha(got), golden[name + "_sha256"])


@pytest.mark.parametrize("c", bc.ENCODE_CASES, ids=[c["name"] for c in bc.ENCODE_CASES])
def test_oracle_matches_the_images_cv2_encoded(golden, c):
    assert np.array_equal(sha(bc.encode_image(c, bo.to_bgr)), golden[c["name"] + ".img_sha256"])


def test_cases_cover_every_layout_and_size_class():
    assert set(bc.LAYOUTS) == set(eng.BAYER_LAYOUTS) and len(eng.BAYER_LAYOUTS) == 8
    for layout in bc.LAYOUTS:
        mine = [c for c in bc.CASES if c[1] == layout]
        assert {(fw % 2, fh % 2) for _, _, _, (fh, fw), _, _, _ in mine} == {(0, 0), (0, 1), (1, 0), (1, 1)}
        assert any(min(hw) == 1 for _, _, _, hw, _, _, _ in mine) and any(min(hw) == 2 for _, _, _, hw, _, _, _ in mine)
        assert any(min(hw) == 3 for _, _, _, hw, _, _, _ in mine) and any(hw == (1080, 1920) for _, _, _, hw, _, _, _ in mine)
        assert any(c[6] is not None for c in mine)
        wins = [(c[5], c[3]) for c in mine if c[5] is not None]
        assert any(x0 == 0 for (x0, _, _, _), _ in wins) and any(y0 == 0 for (_, y0, _, _), _ in wins)
        assert any(x0 + w == fw for (x0, _, w, _), (_, fw) in wins) and any(y0 + h == fh for (_, y0, _, h), (fh, _) in wins)
        assert any(w == h == 1 for (_, _, w, h), _ in wins) and any(x0 % 2 and y0 % 2 for (x0, y0, _, _), _ in wins)
    assert {c["layout"] for c in bc.ENCODE_CASES} == set(bc.LAYOUTS)


def test_oracle_rules_on_a_hand_made_frame():
    """A 4 x 4 RGGB (bayer_bg) frame: the bilinear and edge-aware G at an R site, the diagonal B, a G site's neighbours, the
    border clamp, and frames under 3 pixels on a side."""
    raw = np.array([[10, 20, 30, 40],
                    [50, 60, 70, 80],
                    [90, 100, 110, 120],
                    [130, 140, 150, 160]], np.uint8)
    # (2, 2) is an R site (even row, even column): G from 4 neighbours, B from the diagonals
    bl, ea = bo.to_bgr(raw, "bayer_bg"), bo.to_bgr(raw, "bayer_bg_ea")
    assert tuple(bl[2, 2]) == ((60 + 80 + 140 + 160 + 2) >> 2, (70 + 150 + 100 + 120 + 2) >> 2, 110)
    # |L - R| = 20 <= |U - D| = 80: the edge-aware G is the horizontal mean
    assert tuple(ea[2, 2]) == (bl[2, 2, 0], (100 + 120 + 1) >> 1, 110)
    # (1, 2) is a G site on a blue row: B from left / right, R from up / down
    assert tuple(bl[1, 2]) == ((60 + 80 + 1) >> 1, 70, (30 + 110 + 1) >> 1)
    assert np.array_equal(bl[0], bl[1]) and np.array_equal(bl[:, 3], bl[:, 2]) and np.array_equal(bl[:, 0], bl[:, 1])
    for shape in ((1, 1), (2, 9), (9, 2)):
        assert not bo.to_bgr(np.full(shape, 200, np.uint8), "bayer_rg").any()
    # the mosaic of a converted flat colour gives back the colour at every site
    flat = np.zeros((6, 8, 3), np.uint8)
    flat[...] = (40, 120, 200)
    for layout in bc.LAYOUTS:
        assert (bo.to_bgr(bo.mosaic(flat, layout), layout) == (40, 120, 200)).all(), layout


def bayer(*descs):
    arr = (eng.BayerFrame * len(descs))()
    for a, d in zip(arr, descs):
        (a.data, a.pitch, a.fw, a.fh, a.x0, a.y0, a.w, a.h, a.red_x, a.red_y, a.edge_aware) = d
    return arr


FIELDS = ("data", "pitch", "fw", "fh", "x0", "y0", "w", "h", "red_x", "red_y", "edge_aware")


def test_descriptor_fits_the_encoder_union():
    assert eng.ctypes.sizeof(eng.BayerFrame) <= eng.ctypes.sizeof(eng.Yuv420Frame)
    assert eng.ctypes.sizeof(eng._EncFrame) == eng.ctypes.sizeof(eng.Yuv420Frame)
    assert eng.JPEG_SRC_BAYER == 5 and eng.lib().yfv2_abi_version() == 1


def test_bayer_abi_rejects_bad_descriptors_before_any_launch():
    """Each bad field refused by yfv2_resize_bayer_u8 with its reason, naming the entry and the frame, and by
    yfv2_jpeg_encode_plan wrapped as YFV2_JPEG_SRC_BAYER, naming the output; one in the third launch's chunk too."""
    fake = 0x1000                                              # never dereferenced: every check runs on the host first
    good = (fake, 2048, 1921, 1081, 3, 5, 1900, 1070, 1, 0, 1)
    faults = [(dict(data=None), "null data"), (dict(fw=0), "fw and fh"), (dict(fh=0), "fw and fh"), (dict(fw=-3), "fw and fh"),
              (dict(pitch=1920, fw=1921, x0=0, w=1921), "pitch < fw"), (dict(pitch=-1), "pitch < fw"),
              (dict(w=0), "window"), (dict(h=0), "window"), (dict(w=-1), "window"), (dict(x0=-1), "window"),
              (dict(y0=-1), "window"), (dict(x0=22), "window"), (dict(y0=12), "window"), (dict(w=1919), "window"),
              (dict(x0=1 << 30, w=1 << 30), "window"),
              (dict(red_x=2), "red_x and red_y"), (dict(red_y=-1), "red_x and red_y"),
              (dict(edge_aware=2), "edge_aware"), (dict(edge_aware=-1), "edge_aware")]

    def bad(f):
        d = dict(zip(FIELDS, good))
        d.update(f)
        return tuple(d.values())

    L = eng.lib()
    dst = eng.ctypes.c_void_p(fake)
    assert jc.plan_error(eng.JPEG_SRC_BAYER, "bayer", bayer(good, good))[0] == 0
    for n in (0, -1):
        assert L.yfv2_resize_bayer_u8(bayer(good), n, 352, 352, dst, None) == -1
        assert b"resize_bayer_u8: null frames / dst or N <= 0" in L.yfv2_last_error()
    assert L.yfv2_resize_bayer_u8(bayer(good), 1, 352, 352, None, None) == -1
    for H, W in ((0, 352), (352, 0), (32769, 352), (352, 32769)):
        assert L.yfv2_resize_bayer_u8(bayer(good), 1, H, W, dst, None) == -1
        assert b"resize_bayer_u8: target" in L.yfv2_last_error()
    for f, why in faults:
        assert L.yfv2_resize_bayer_u8(bayer(good, bad(f)), 2, 352, 352, dst, None) == -1, f
        err = L.yfv2_last_error()
        assert b"resize_bayer_u8: frame 1: " + why.encode() in err, (f, err)
        rc, err = jc.plan_error(eng.JPEG_SRC_BAYER, "bayer", bayer(good, bad(f)))
        assert rc == -1 and b"jpeg_encode_plan: output 1: frame: " + why.encode() in err, (f, err)
    assert L.yfv2_resize_bayer_u8(bayer(*([good] * 130 + [bad(faults[0][0])])), 131, 352, 352, dst, None) == -1
    assert b"frame 130: null data" in L.yfv2_last_error()


def test_encode_plan_keeps_regions_inside_the_window():
    """An output's region is a region of the descriptor's window (w x h), not of the whole frame."""
    fake = 0x1000
    srcs = (eng.JpegEncSrc * 1)()
    s = srcs[0]
    s.kind = eng.JPEG_SRC_BAYER
    s.f.bayer = bayer((fake, 640, 640, 480, 100, 50, 200, 100, 0, 0, 0))[0]
    L = eng.lib()
    mb, wb, ab = eng.ctypes.c_size_t(), eng.ctypes.c_size_t(), eng.ctypes.c_size_t()
    for (x0, y0, w, h), ok in [((0, 0, 200, 100), True), ((199, 99, 1, 1), True), ((0, 0, 201, 100), False),
                               ((150, 0, 51, 10), False), ((0, 60, 10, 41), False)]:
        s.x0, s.y0, s.w, s.h = x0, y0, w, h
        rc = L.yfv2_jpeg_encode_plan(srcs, 1, None, 0, eng.ctypes.byref(mb), eng.ctypes.byref(wb), None, eng.ctypes.byref(ab))
        assert (rc == 0) == ok, ((x0, y0, w, h), L.yfv2_last_error())
        if not ok:
            assert b"outside the 200x100 frame" in L.yfv2_last_error()


def test_python_entries_refuse_bad_frames_before_anything_runs():
    raw = np.zeros((48, 64), np.uint8)
    win = eng.BayerWindow(raw, 3, 5, 20, 10)
    cases = [
        ([raw], "bayer", "layout"), ([raw], "bayer_bggr", "layout"), ([raw], "BAYER_BG", "layout"), ([raw], "bayer_bg_vng", "layout"),
        ([raw], ["bayer_bg", "bayer"], "layout"),
        ([raw.astype(np.uint16)], "bayer_bg", "uint8"), ([torch.zeros((48, 64), dtype=torch.int16)], "bayer_gr", "uint8"),
        ([np.zeros((48, 64, 1), np.uint8)], "bayer_rg", "2-D"), ([raw[None]], "bayer_gb_ea", "2-D"), ([raw[0]], "bayer_bg", "2-D"),
        ([np.zeros((0, 64), np.uint8)], "bayer_bg", "h, w > 0"), ([np.zeros((48, 0), np.uint8)], "bayer_rg_ea", "h, w > 0"),
        ([eng.BayerWindow(raw, 0, 0, 65, 48)], "bayer_bg", "not inside"), ([eng.BayerWindow(raw, -1, 0, 2, 2)], "bayer_bg", "not inside"),
        ([eng.BayerWindow(raw, 63, 47, 2, 1)], "bayer_bg", "not inside"), ([eng.BayerWindow(raw, 5, 5, 0, 3)], "bayer_bg", "not inside"),
        ([eng.BayerWindow(raw.astype(np.int8), 0, 0, 2, 2)], "bayer_bg", "uint8"),
        ([win], "bgr", r"\[h, w, 3\]"), ([win], "gray", "uint8"),
        # a bad frame after good ones of other kinds: nothing is launched for the good ones either (no device is touched)
        ([np.zeros((48, 64, 3), np.uint8), raw, win, np.zeros((72, 64), np.uint8), raw.astype(np.float32)],
         ["bgr", "bayer_bg", "bayer_gr_ea", "nv12", "bayer_rg"], "frame 4"),
    ]
    entries = {"resize_frames": lambda frames, layout: eng.resize_frames(frames, 352, 352, layout, device="cuda:0"),
               "encode_jpeg": lambda frames, layout: eng.encode_jpeg(frames, layout=layout, device="cuda:0"),
               "crop_frame": lambda frames, layout: eng.crop_frame(frames[0], layout, 0, 0, 2, 2)}
    for frames, layout, msg in cases:
        for name, call in entries.items():
            if name == "crop_frame" and (len(frames) != 1 or not isinstance(layout, str)):
                continue
            with pytest.raises(eng.Yfv2Error, match=msg) as e:
                call(frames, layout)
            assert str(e.value).startswith(name + ": "), (layout, str(e.value))


def test_crop_frame_windows_compose_and_stay_inside():
    raw = np.arange(48 * 64, dtype=np.int64).astype(np.uint8).reshape(48, 64)
    w1 = eng.crop_frame(raw, "bayer_gb", 5, 7, 40, 30)
    assert isinstance(w1, eng.BayerWindow) and (w1.x0, w1.y0, w1.w, w1.h) == (5, 7, 40, 30)
    assert tuple(w1.raw.shape) == (48, 64) and w1.raw.data_ptr() == raw.ctypes.data      # the whole frame, not copied
    w2 = eng.crop_frame(w1, "bayer_gb", 3, 1, 37, 29)
    assert (w2.x0, w2.y0, w2.w, w2.h) == (8, 8, 37, 29) and w2.raw.data_ptr() == raw.ctypes.data
    assert eng.frame_size(w2, "bayer_gb") == (29, 37) and eng.frame_size(raw, "bayer_gb_ea") == (48, 64)
    assert eng.frame_size(torch.from_numpy(raw)[:, 1:], "bayer_rg") == (48, 63)
    w3 = eng.crop_frame(w2, "bayer_gb", 36, 28, 1, 1)                                    # odd offsets need no alignment
    assert (w3.x0, w3.y0, w3.w, w3.h) == (44, 36, 1, 1) and eng.frame_size(w3, "bayer_gb") == (1, 1)
    for x0, y0, w, h in [(0, 0, 38, 29), (0, 0, 37, 30), (1, 0, 37, 29), (0, -1, 5, 5), (0, 0, 0, 1)]:
        with pytest.raises(eng.Yfv2Error, match="crop_frame: window .* is not inside the 37x29 frame"):
            eng.crop_frame(w2, "bayer_gb", x0, y0, w, h)
    # what the oracle says the window is: the crop of the converted WHOLE frame, not the conversion of the cropped raw
    whole = bo.to_bgr(raw, "bayer_gb")
    assert np.array_equal(bo.window_bgr(raw, "bayer_gb", 8, 8, 37, 29), whole[8:37, 8:45])
    assert not np.array_equal(bo.to_bgr(raw[8:37, 8:45], "bayer_gb"), whole[8:37, 8:45])


def test_tile_regions_are_not_rounded_for_bayer():
    from utils import frames as uf
    for layout in eng.BAYER_LAYOUTS:
        tiles = uf.tile_regions(1921, 1081, 3, 2, 0.2, True, layout)
        assert tiles == uf.tile_regions(1921, 1081, 3, 2, 0.2, True, "bgr")
        assert any(x0 % 2 or w % 2 for x0, _, w, _ in tiles[1:])

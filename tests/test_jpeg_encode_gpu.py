"""The device JPEG encode (yfv2_jpeg_encode) against cv2.imencode's bytes frozen in tests/golden/jpeg_encode_cases.npz: every
case in one mixed call and one call per output, a batch of 256 full-HD frames against batch 1, the round trip through the
project's decoder against cv2.imdecode's frames, and the crops of detections."""
import hashlib
import os

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import jpeg_encode_cases as C
import yfv2_engine as eng

pytestmark = pytest.mark.gpu
GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(GOLDEN_DIR, "jpeg_encode_cases.npz")))


@pytest.fixture(scope="module")
def photos():
    names = ("000004.jpg", "000139.jpg")
    files = [open(os.path.join(GOLDEN_DIR, n), "rb").read() for n in names]
    return dict(zip(names, eng.decode_jpeg(files)))


def _frame(c, photos):
    return (photos[c["photo"]], "bgr") if c["photo"] else (C.frame(c["layout"], c["w"], c["h"], c["kind"], c["seed"]), c["layout"])


def _matches(c, b, golden):
    if c["name"] in golden:
        return b == golden[c["name"]].tobytes()
    return len(b) == int(golden[c["name"] + ".len"]) and hashlib.sha256(b).digest() == golden[c["name"] + ".sha"].tobytes()


def _encode(cs, photos):
    frames, layouts, regions = [], [], []
    for k, c in enumerate(cs):
        f, lay = _frame(c, photos)
        frames.append(f)
        layouts.append(lay)
        regions.append((k,) + tuple(c["region"]) if c["region"] else (k, 0, 0, None, None))
    return eng.encode_jpeg(frames, quality=[c["quality"] for c in cs], sampling=[c["sampling"] for c in cs],
                           restart_interval=[c["restart"] for c in cs], layout=layouts, regions=regions)


def test_every_case_in_one_call(golden, photos):
    cs = C.cases()
    got = _encode(cs, photos)
    bad = [c["name"] for c, b in zip(cs, got) if not _matches(c, b, golden)]
    assert not bad, bad


def test_one_call_per_output_equals_the_mixed_call(golden, photos):
    cs = [c for c in C.cases() if c["w"] * c["h"] <= 352 * 352][::3]
    mixed = _encode(cs, photos)
    for c, b in zip(cs, mixed):
        assert _encode([c], photos)[0] == b, c["name"]


def test_shared_frame_regions(golden):
    """Several outputs of one frame: every region of a case's frame in one call"""
    cs = [c for c in C.cases() if c["name"].startswith("region_") and c["layout"] == "nv12"]
    f = C.frame("nv12", 64, 48, "noise", 0)
    got = eng.encode_jpeg([f], quality=95, sampling=[c["sampling"] for c in cs], layout="nv12",
                          regions=[(0,) + tuple(c["region"]) for c in cs])
    for c, b in zip(cs, got):
        assert _matches(c, b, golden), c["name"]


def test_batch_of_256_full_hd_frames_equals_batch_1():
    rng = np.random.RandomState(5)
    base = [rng.randint(0, 256, (1080, 1920, 3), np.uint8) for _ in range(3)]
    base.append(np.ascontiguousarray(np.repeat(np.repeat(rng.randint(0, 256, (135, 240, 3), np.uint8), 8, 0), 8, 1)))
    dev = [torch.from_numpy(b).cuda() for b in base]
    one = [eng.encode_jpeg([d])[0] for d in dev]
    got = eng.encode_jpeg([dev[i % 4] for i in range(256)])
    assert all(got[i] == one[i % 4] for i in range(256))


def test_round_trip_through_the_decoder(golden, photos):
    cs = [c for c in C.cases() if c["name"] in C.ROUNDTRIP]
    files = _encode(cs, photos)
    frames = eng.decode_jpeg(files)
    for c, f in zip(cs, frames):
        assert hashlib.sha256(f.cpu().numpy().tobytes()).digest() == golden[c["name"] + ".decoded"].tobytes(), c["name"]


def test_device_out_matches_bytes():
    f = C.frame("bgr", 37, 53, "noise", 0)
    arena, offsets, lengths = eng.encode_jpeg([f, f], quality=[95, 10], device_out=True)
    want = eng.encode_jpeg([f, f], quality=[95, 10])
    lens = lengths.cpu().numpy()
    for k in range(2):
        assert arena[int(offsets[k]):int(offsets[k]) + int(lens[k])].cpu().numpy().tobytes() == want[k]


def test_encode_detections_are_the_crops(photos):
    import utils.frames as uf
    frames = [photos[n] for n in ("000004.jpg", "000139.jpg")]
    rows = [torch.tensor([[10.4, 20.6, 120.2, 200.9, 0.9, 0], [-5.0, -3.0, 30.0, 40.0, 0.8, 1], [300.0, 200.0, 9000.0, 9000.0, 0.7, 2]]),
            torch.tensor([[50.0, 60.0, 51.0, 61.0, 0.5, 3]])]
    got = uf.encode_detections(frames, rows, quality=90)
    for f, r, g in zip(frames, rows, got):
        h, w = f.shape[:2]
        assert len(g) == len(r)
        for reg, b in zip(uf.detection_regions(r, h, w), g):
            assert b == eng.encode_jpeg([f], quality=90, regions=[(0,) + reg])[0]
    assert uf.detection_regions(rows[0], 500, 353) == [(10, 20, 110, 180), (0, 0, 30, 40), (300, 200, 53, 300)]


def test_refusals_raise_before_launch():
    f = C.frame("bgr", 16, 16, "noise", 0)
    for kw in (dict(params=[eng.IMWRITE_JPEG_OPTIMIZE, 1]), dict(params=[eng.IMWRITE_JPEG_PROGRESSIVE, 1]),
               dict(params=[eng.IMWRITE_JPEG_LUMA_QUALITY, 50]), dict(sampling="440"), dict(regions=[(0, 10, 10, 7, 0)]),
               dict(regions=[(0, 10, 10, 7, 7)])):
        with pytest.raises(eng.Yfv2Error, match="output 0"):
            eng.encode_jpeg([f], **kw)

"""JPEG files decoded on the device (decode_jpeg: yfv2_jpeg_parse + yfv2_jpeg_decode) against cv2.imdecode's frozen bytes, one file
per call and every fixture in one batch; read_images and detect_files on the reference's photos; the arena's frames fed to the
resize in place; unsupported files refused before anything is launched."""
import os

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import jpeg_cases as jc
import synth
import yfv2_engine as eng

pytestmark = pytest.mark.gpu

PHOTOS = ("000139", "000004")


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "jpeg_cases.npz"))


def modelzoo_detector(golden_dir):
    import model.detector as det
    w = synth.load_modelzoo_weights(golden_dir)
    m = det.Detector(80, 3, True)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
    return m.cuda().eval()


def test_every_fixture_one_file_per_call(golden):
    bad = []
    for case in jc.CASES:
        name = case[0]
        (got,) = eng.decode_jpeg([golden["jpg_" + name]], "cuda")
        if not jc.equals_golden(golden, name, got.cpu().numpy()):
            bad.append(name)
    assert not bad, "differ from cv2: %s" % bad


def test_every_fixture_in_one_batch(golden):
    names = [c[0] for c in jc.CASES]
    order = list(range(len(names)))
    np.random.RandomState(3).shuffle(order)                  # sizes, samplings and restart counts interleaved in the arena
    got = eng.decode_jpeg([golden["jpg_" + names[i]] for i in order], "cuda")
    for i, g in zip(order, got):
        assert g.is_cuda and g.dtype == torch.uint8
        assert jc.equals_golden(golden, names[i], g.cpu().numpy()), names[i]


def test_read_images_equals_cv2_imread_of_the_reference_photos(golden_dir):
    frames = np.load(os.path.join(golden_dir, "frames_modelzoo.npz"))
    got = __import__("utils.frames", fromlist=["read_images"]).read_images([os.path.join(golden_dir, s + ".jpg") for s in PHOTOS])
    for s, g in zip(PHOTOS, got):
        assert np.array_equal(g.cpu().numpy(), frames[s]), s


def test_detect_files_equals_detect_frames_on_the_golden_frames(golden_dir):
    import utils.frames as uf
    frames = np.load(os.path.join(golden_dir, "frames_modelzoo.npz"))
    m = modelzoo_detector(golden_dir)
    cfg = synth.coco_cfg()
    got = uf.detect_files(m, [os.path.join(golden_dir, s + ".jpg") for s in PHOTOS], cfg, conf_thres=0.3, iou_thres=0.4)
    want = uf.detect_frames(m, [frames[s] for s in PHOTOS], cfg, conf_thres=0.3, iou_thres=0.4)
    assert len(got) == len(want) == 2
    for g, w in zip(got, want):
        assert g.shape[0] > 0 and torch.equal(g, w)


def test_arena_frames_feed_the_resize_in_place(golden, golden_dir):
    frames = np.load(os.path.join(golden_dir, "frames_modelzoo.npz"))
    files = [np.fromfile(os.path.join(golden_dir, s + ".jpg"), np.uint8) for s in PHOTOS]
    extra = ["exif6_II", "size333x500_411", "fullhd_420"]
    files += [golden["jpg_" + n] for n in extra]
    got = eng.decode_jpeg(files, "cuda")
    for n, g in zip(extra, got[2:]):
        assert jc.equals_golden(golden, n, g.cpu().numpy()), n               # so these are cv2's frames
    wants = [frames[s] for s in PHOTOS] + [g.cpu().numpy() for g in got[2:]]
    base = got[0].untyped_storage().data_ptr()
    assert all(g.untyped_storage().data_ptr() == base for g in got)       # views into one arena, no copies
    for H, W in ((352, 352), (96, 160)):
        assert torch.equal(eng.resize_bgr(got, W, H), eng.resize_bgr(wants, W, H, device="cuda"))


def test_unsupported_files_raise_before_any_launch(golden):
    good = golden["jpg_q75_420_opt0"]
    for name, _, reason in jc.UNSUPPORTED:
        if name == "cut_header":
            continue                                          # malformed files stay with the CPU tests
        torch.cuda.synchronize()
        with pytest.raises(eng.Yfv2Error, match=r"b\.jpg: .*%s" % reason):
            eng.decode_jpeg([good, golden["bad_" + name]], "cuda", names=["a.jpg", "b.jpg"])
    # the refusal happens in the host parse: nothing was allocated on the device for the batch
    before = torch.cuda.memory_allocated()
    with pytest.raises(eng.Yfv2Error, match="progressive"):
        eng.decode_jpeg([good, golden["bad_progressive"]], "cuda")
    assert torch.cuda.memory_allocated() == before


def test_phases_run_separately_give_the_same_frames(golden):
    files = [golden["jpg_" + c[0]] for c in jc.CASES[:40]]
    b = eng.JpegBatch(files, "cuda")
    for ph in (eng.JPEG_ENTROPY, eng.JPEG_IDCT, eng.JPEG_COLOR):
        b.decode(ph)
    b.check()
    for c, g in zip(jc.CASES[:40], b.frames()):
        assert jc.equals_golden(golden, c[0], g.cpu().numpy()), c[0]

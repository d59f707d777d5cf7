"""Progressive JPEG files (tests/jpeg_progressive_cases.py) decoded on the device (JpegBatch(progressive=True)), one file per call
and in a shuffled batch mixed with the jpeg_cases and jpeg_foreign fixtures.  On every accepted file, damaged ones included, the
device's bytes and flags equal the CPU build of the same functions (tests/jpeg_progressive_harness.cu); on unflagged files the
bytes are cv2's.  read_images / detect_files(progressive=True) on the reference's photos re-coded losslessly as progressive
files, against their golden frames; the arena fed to the resize; the flag's default."""
import os

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import jpeg_cases as jc
import jpeg_foreign_cases as fc
import jpeg_progressive_cases as pc
import yfv2_engine as eng
from test_jpeg_progressive_cpu import harness, run_harness  # noqa: F401  (the harness fixture)

pytestmark = pytest.mark.gpu

ACCEPTED = [n for n in pc.CASES if n not in pc.REFUSED]


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "jpeg_progressive.npz"))


@pytest.fixture(scope="module")
def host(golden, harness):  # noqa: F811
    """name -> (flags, BGR bytes) of the CPU build"""
    items = [(n, golden["jpg_" + n]) for n in ACCEPTED]
    results, outs = run_harness(harness, items)
    out = {}
    for (name, _), (status, w, h, err, _, _), path in zip(items, results, outs):
        assert status == 0, name
        out[name] = (err, np.fromfile(path, np.uint8).reshape(h, w, 3))
    return out


def device_decode(files, phases=None):
    b = eng.JpegBatch(files, "cuda", progressive=True)
    for ph in phases or (eng.JPEG_ALL,):
        b.decode(ph)
    return [f.cpu().numpy() for f in b.frames()], b.errors.cpu().tolist()


def check(golden, host, name, got, err, bad):
    herr, hbytes = host[name]
    if err != herr or not np.array_equal(got, hbytes):
        bad.append((name, "device != host build", err, herr))
    elif not err and "none_" + name in golden.files:
        bad.append((name, "cv2 cannot decode it, not flagged"))
    elif not err and not jc.equals_golden(golden, name, got):
        bad.append((name, "unflagged, differs from cv2"))
    elif err and name not in pc.DAMAGED:
        bad.append((name, "flagged though undamaged", err))


def test_every_case_one_file_per_call(golden, host):
    bad = []
    for name in ACCEPTED:
        (got,), (err,) = device_decode([golden["jpg_" + name]])
        check(golden, host, name, got, err, bad)
    assert not bad, bad


def test_mixed_batch_with_the_baseline_fixtures(golden, golden_dir, host):
    base = np.load(os.path.join(golden_dir, "jpeg_cases.npz"))
    foreign = np.load(os.path.join(golden_dir, "jpeg_foreign.npz"))
    files = [("p", n) for n in ACCEPTED] + [("c", c[0]) for c in jc.CASES]
    files += [("f", n) for n in fc.CASES if n not in fc.REFUSED and n not in fc.DAMAGED and "none_" + n not in foreign.files]
    np.random.RandomState(11).shuffle(files)
    src = {"p": golden, "c": base, "f": foreign}
    got, errs = device_decode([src[k]["jpg_" + n] for k, n in files])
    bad = []
    for (kind, name), g, e in zip(files, got, errs):
        if kind == "p":
            check(golden, host, name, g, e, bad)
        elif e or not jc.equals_golden(src[kind], name, g):
            bad.append((name, e))
    assert not bad, bad


def test_phases_run_separately_give_the_same_frames(golden, host):
    names = [n for n in ACCEPTED if n.startswith(("script_", "cv2_q", "enc_"))]
    got, errs = device_decode([golden["jpg_" + n] for n in names], (eng.JPEG_ENTROPY, eng.JPEG_IDCT, eng.JPEG_COLOR))
    bad = []
    for n, g, e in zip(names, got, errs):
        check(golden, host, n, g, e, bad)
    assert not bad, bad


def test_a_batch_of_progressive_files_only(golden):
    names = [n for n in ACCEPTED if n.startswith("cv2_") and "none_" + n not in golden.files]
    got = eng.decode_jpeg([golden["jpg_" + n] for n in names], "cuda", progressive=True)
    for n, g in zip(names, got):
        assert jc.equals_golden(golden, n, g.cpu().numpy()), n


@pytest.mark.parametrize("script", ["cv2", "seeded"])
def test_read_images_and_detect_files_on_the_recoded_photos(golden, golden_dir, tmp_path, script):
    import synth
    import utils.frames as uf
    from test_jpeg_gpu import modelzoo_detector
    frames = np.load(os.path.join(golden_dir, "frames_modelzoo.npz"))
    paths = []
    for s in pc.PHOTOS:
        paths.append(str(tmp_path / ("tx_%s_%s.jpg" % (script, s))))
        golden["jpg_tx_%s_%s" % (script, s)].tofile(paths[-1])
    want = [torch.from_numpy(frames[s]).cuda() for s in pc.PHOTOS]
    got = uf.read_images(paths, progressive=True)
    for s, g, w in zip(pc.PHOTOS, got, want):
        assert torch.equal(g, w), s
    with pytest.raises(eng.Yfv2Error, match="progressive DCT"):
        uf.read_images(paths)
    m = modelzoo_detector(golden_dir)
    cfg = synth.coco_cfg()
    dets = uf.detect_files(m, paths, cfg, conf_thres=0.3, iou_thres=0.4, progressive=True)
    ref = uf.detect_frames(m, [frames[s] for s in pc.PHOTOS], cfg, conf_thres=0.3, iou_thres=0.4)
    assert len(dets) == len(ref) == 2
    for d, r in zip(dets, ref):
        assert d.shape[0] > 0 and torch.equal(d, r)


def test_arena_frames_feed_the_resize_in_place(golden):
    names = ["tx_seeded_000004", "cv2_fullhd_420", "cv2_exif6_II", "script_420_3", "pil_sub2_q50"]
    got = eng.decode_jpeg([golden["jpg_" + n] for n in names], "cuda", progressive=True)
    wants = []
    for n, g in zip(names, got):
        assert jc.equals_golden(golden, n, g.cpu().numpy()), n
        wants.append(g.cpu().numpy())
    base = got[0].untyped_storage().data_ptr()
    assert all(g.untyped_storage().data_ptr() == base for g in got)
    for H, W in ((352, 352), (96, 160)):
        assert torch.equal(eng.resize_bgr(got, W, H), eng.resize_bgr(wants, W, H, device="cuda"))


def test_without_the_flag_decode_jpeg_raises_before_any_allocation(golden, golden_dir):
    good = np.load(os.path.join(golden_dir, "jpeg_cases.npz"))["jpg_q75_420_opt0"]
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    with pytest.raises(eng.Yfv2Error, match=r"b\.jpg: progressive DCT \(SOF2\)"):
        eng.decode_jpeg([good, golden["jpg_cv2_q50_420"]], "cuda", names=["a.jpg", "b.jpg"])
    assert torch.cuda.memory_allocated() == before


def test_a_cut_file_raises_as_cut_short(golden):
    with pytest.raises(eng.Yfv2Error, match=r"b\.jpg: entropy-coded data ran out"):
        eng.decode_jpeg([golden["jpg_enc_base"], golden["jpg_cut_eoi_d9"]], "cuda", names=["a.jpg", "b.jpg"], progressive=True)

"""Image files into training and evaluation batches on the GPU: yfv2_jpeg_decode_resize against decode + resize_bgr on every JPEG
fixture, DeviceLoader against the reference's own TensorDataset(imgaug=False) + collate_fn (tests/golden/loader_cases.npz), and
train_dist.py --device-decode / evaluation() fed by the device loader."""
import os

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import jpeg_cases as jc
import jpeg_progressive_cases as jpc
import loader_cases as lc
import synth

pytestmark = pytest.mark.gpu

# (W, H): the network input, a non-square one, an upscale past every fixture (1080p included), a 1-pixel-wide target
SIZES = [(352, 352), (320, 192), (2048, 1152), (1, 5)]


@pytest.fixture(scope="module")
def golden(golden_dir):
    return lc.load(golden_dir)


@pytest.fixture()
def dataset(golden, golden_dir, tmp_path, monkeypatch):
    z, names = golden
    files = lc.build(str(tmp_path), names, golden_dir, z)
    monkeypatch.chdir(tmp_path)
    return z, names, files


def _fused_vs_two_calls(files, progressive, W, H):
    import yfv2_engine as eng
    b = eng.JpegBatch(files, "cuda", progressive=progressive)
    b.decode()
    frames = b.frames()
    flags = b.flags()
    want = eng.resize_bgr(frames, W, H)
    got = torch.full((len(files), 3, H, W), 7, dtype=torch.uint8, device="cuda")
    f = eng.JpegBatch(files, "cuda", progressive=progressive)
    f.decode_resize(got, W, H)
    assert f.flags() == flags
    return got, want, flags


@pytest.mark.parametrize("W,H", SIZES, ids=["%dx%d" % s for s in SIZES])
def test_decode_resize_equals_decode_then_resize_baseline(golden_dir, W, H):
    z = np.load(os.path.join(golden_dir, "jpeg_cases.npz"))
    files = [z["jpg_" + c[0]] for c in jc.CASES] + [z["cut_" + jc.TRUNCATED_SCAN]]
    got, want, flags = _fused_vs_two_calls(files, False, W, H)
    assert flags[:-1] == [0] * len(jc.CASES) and flags[-1] & 1
    for i, c in enumerate(jc.CASES + [("cut",)]):
        assert torch.equal(got[i], want[i]), c[0]


@pytest.mark.parametrize("W,H", SIZES, ids=["%dx%d" % s for s in SIZES])
def test_decode_resize_equals_decode_then_resize_progressive(golden_dir, W, H):
    z = np.load(os.path.join(golden_dir, "jpeg_progressive.npz"))
    names = [n for n in jpc.CASES if n not in jpc.REFUSED]
    got, want, flags = _fused_vs_two_calls([z["jpg_" + n] for n in names], True, W, H)
    for i, n in enumerate(names):
        assert bool(flags[i]) == (n in jpc.DAMAGED), n
        if not flags[i]:                  # a flagged frame (a run past its band) is not promised to be the same twice
            assert torch.equal(got[i], want[i]), n


def test_decode_resize_jpeg_matches_the_reference_photos_and_refuses_as_decode_jpeg(golden_dir):
    import yfv2_engine as eng
    g = np.load(os.path.join(golden_dir, "images_modelzoo.npz"))
    files = []
    for p in lc.PHOTOS:
        with open(os.path.join(golden_dir, p + ".jpg"), "rb") as f:
            files.append(f.read())
    out = torch.empty((2, 3, 352, 352), dtype=torch.uint8, device="cuda")
    assert eng.decode_resize_jpeg(files, 352, 352, out=out) is out
    for i, p in enumerate(lc.PHOTOS):
        assert np.array_equal(out[i].cpu().numpy(), g[p + "_u8"][0]), p
    z = np.load(os.path.join(golden_dir, "jpeg_cases.npz"))
    with pytest.raises(eng.Yfv2Error, match=r"1 of 2 files refused: b\.png"):
        eng.decode_resize_jpeg([files[0], z["bad_png"]], 352, 352, names=["a.jpg", "b.png"])
    with pytest.raises(eng.Yfv2Error, match="failed to decode: cut"):
        eng.decode_resize_jpeg([z["cut_" + jc.TRUNCATED_SCAN]], 352, 352, names=["cut"])
    with pytest.raises(eng.Yfv2Error, match="out must be"):
        eng.decode_resize_jpeg(files, 352, 352, out=torch.empty((2, 3, 352, 351), dtype=torch.uint8, device="cuda"))


def test_decode_resize_equals_the_reference_items(dataset):
    """Every file the device decodes without a flag, straight against TensorDataset(imgaug=False)'s recorded bytes."""
    import yfv2_engine as eng
    z, names, files = dataset
    infos = eng.parse_jpeg([files[n] for n in names], progressive=True, strict=False)[0]
    idx = [i for i, inf in enumerate(infos) if inf["status"] == 0]
    for (W, H) in lc.SIZES:
        b = eng.JpegBatch([files[names[i]] for i in idx], "cuda", progressive=True)
        out = b.decode_resize(torch.empty((len(idx), 3, H, W), dtype=torch.uint8, device="cuda"), W, H)
        flags = b.flags()
        want = z["sha_%dx%d" % (W, H)]
        checked = 0
        for k, i in enumerate(idx):
            if flags[k]:
                assert names[i].split("/")[0] in ("cut", "pdamaged"), names[i]
                continue
            assert bytes(lc.digest(out[k].cpu().numpy())) == bytes(want[i]), (names[i], W, H)
            checked += 1
        assert checked >= len(jc.CASES) + len(lc.PROG) + len(lc.PHOTOS)


def _loader(z, W, H, B, workers):
    from utils.device_data import device_loader
    return device_loader(lc.LIST, W, H, B, torch.device("cuda"), num_workers=workers, fallback=lc.fallback_reader(z))


@pytest.mark.parametrize("workers", [0, 2])
@pytest.mark.parametrize("B", lc.BATCHES)
def test_device_loader_equals_the_reference_batches(dataset, workers, B):
    z, names, _ = dataset
    W, H = lc.SIZES[0]
    shas, tshas, sizes = z["sha_%dx%d" % (W, H)], z["targets_b%d" % B], []
    dl = _loader(z, W, H, B, workers)
    assert len(dl) == len(tshas) > 2 and len(names) % B
    for k, (imgs, targets) in enumerate(dl):
        assert imgs.is_cuda and imgs.dtype == torch.uint8 and tuple(imgs.shape[1:]) == (3, H, W)
        sizes.append(imgs.shape[0])
        host = imgs.cpu().numpy()          # on the current stream, which the loader made wait for the side stream
        for j in range(imgs.shape[0]):
            assert bytes(lc.digest(host[j])) == bytes(shas[k * B + j]), names[k * B + j]
        assert not targets.is_cuda and bytes(lc.digest(targets.numpy())) == bytes(tshas[k]), k
    assert sizes == [B] * (len(names) // B) + [len(names) % B]


def test_device_loader_at_a_non_square_size_while_the_consumer_writes_its_batches(dataset):
    """Each batch is overwritten on the current stream right after it is checked, as the in-place device augmentation does, while
    the next one is decoded on the side stream."""
    z, names, _ = dataset
    W, H = lc.SIZES[1]
    shas = z["sha_%dx%d" % (W, H)]
    n = 0
    for imgs, _ in _loader(z, W, H, 16, 2):
        got = [bytes(lc.digest(im)) for im in imgs.cpu().numpy()]
        assert got == [bytes(s) for s in shas[n:n + len(got)]]
        imgs.fill_(0)
        n += len(got)
    assert n == len(names)


DATA = ("[name]\nmodel_name=coco\n\n[train-configure]\nepochs=1\nsteps=150,250\nbatch_size=8\nsubdivisions=1\nlearning_rate=0.001\n\n"
        "[model-configure]\npre_weights=%s\nclasses=80\nwidth=352\nheight=352\nanchor_num=3\n"
        "anchors=12.64,19.39, 37.88,51.48, 55.71,138.31, 126.91,78.23, 131.57,214.55, 279.92,258.87\n\n"
        "[data-configure]\ntrain=%s\nval=%s\nnames=coco.names\n")


def _device_list(names, path):
    """The files the device decodes without a flag (cv2 need not be installed where this runs)."""
    keep = [n for n in names if n.split("/")[0] in ("base", "prog", "photos")]
    with open(path, "w") as f:
        f.write("".join(n + "\n" for n in keep))
    return keep


def test_train_dist_device_decode_runs(dataset, tmp_path, golden_dir):
    import train_dist
    z, names, _ = dataset
    keep = _device_list(names, "dev.txt")
    torch.save({k: torch.from_numpy(v) for k, v in synth.load_modelzoo_weights(golden_dir).items()}, "w.pth")
    with open("coco.data", "w") as f:
        f.write(DATA % ("w.pth", "dev.txt", "dev.txt"))
    before = {k: v.clone() for k, v in torch.load("w.pth").items()}
    net = train_dist.main(["--data", "coco.data", "--device-decode", "--device-aug", "--max-iters", "4", "--save-dir", str(tmp_path)])
    assert len(keep) >= 32
    after = net.state_dict()
    assert all(torch.isfinite(v.float()).all() for v in after.values())
    assert any(not torch.equal(after[k].cpu(), before[k]) for k in before if k in after)
    with pytest.raises(SystemExit):
        train_dist.main(["--data", "coco.data", "--device-decode", "--max-iters", "1"])


def test_evaluation_fed_by_the_device_loader(dataset, golden_dir):
    """evaluation() over DeviceLoader batches, against evaluation() over the same files as batches of resize_bgr(decode_jpeg)
    + the recorded cv2 frames of the fallback files, whose bytes are checked against the reference's items first."""
    import model.detector
    import utils.utils
    import yfv2_engine as eng
    from utils.device_data import read_labels, label_path, collate_targets
    z, names, files = dataset
    cfg = utils.utils.load_datafile(_write_data(golden_dir))
    read = lc.fallback_reader(z)
    infos = eng.parse_jpeg([files[n] for n in names], progressive=True, strict=False)[0]
    B, shas, ref = 16, z["sha_352x352"], []
    for k in range(0, len(names), B):
        chunk = names[k:k + B]
        frames = []
        for j, n in enumerate(chunk):
            if infos[k + j]["status"] or n.split("/")[0] in ("cut", "pdamaged"):
                frames.append(read(files[n]))
            else:
                frames.append(eng.decode_jpeg([files[n]], progressive=True)[0])
        imgs = eng.resize_bgr(frames, 352, 352)
        for j in range(len(chunk)):
            assert bytes(lc.digest(imgs[j].cpu().numpy())) == bytes(shas[k + j]), chunk[j]
        ref.append((imgs, collate_targets([read_labels(label_path(n)) for n in chunk])))
    device = torch.device("cuda")
    m = model.detector.Detector(80, 3, True)
    m.load_state_dict({kk: torch.from_numpy(v) for kk, v in synth.load_modelzoo_weights(golden_dir).items()})
    m = m.to(device).eval()
    for conf in (0.01, 0.3):
        want = utils.utils.evaluation([(i, t.clone()) for i, t in ref], cfg, m, device, conf)
        got = utils.utils.evaluation(_loader(z, 352, 352, B, 2), cfg, m, device, conf)
        assert want is not None and [float(v) for v in got] == [float(v) for v in want], conf


def _write_data(golden_dir):
    with open("coco.data", "w") as f:
        f.write(DATA % ("None", lc.LIST, lc.LIST))
    return "coco.data"

"""yfv2_aug_geometric on the device (load_mosaic -> random_perspective with border 114 -> fliplr): byte-identical to cv2's goldens
(tests/golden/geom_cases.npz) and to the CPU restatement (tests/geom_oracle.py) on full training batches over several descriptor
chunks, odd sizes and unaligned bases; the labels moved with the pixels; and the trainer with --device-aug-geom."""
import hashlib
import os
import random

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import geom_cases as gc
import geom_oracle as go

pytestmark = pytest.mark.gpu


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest()


@pytest.fixture(scope="module")
def g(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "geom_cases.npz")))


@pytest.mark.parametrize("case", gc.CASES, ids=[c[0] for c in gc.CASES])
def test_device_equals_cv2(g, case):
    import yfv2_engine as eng
    name, N, H, W, seed = case[:5]
    x = torch.from_numpy(gc.images(name, N, H, W, seed, g["jpeg_imgs"])).cuda()
    got = eng.augment_geometric(x, gc.unpack(g[name + "_M"], g[name + "_meta"], g[name + "_s"])).cpu().numpy()
    assert sha(got) == g[name + "_sha256"].tobytes(), name


def mixed_draws(N, H, W, seed, mosaic=0.5):
    """YOLOv5-style draws, half of them mosaics, every third image warped in perspective, flips at random."""
    import utils.device_aug as da
    d = da.draw_geometric(N, H, W, random.Random(seed), mosaic=mosaic, degrees=10, translate=0.1, scale=0.5, shear=5,
                          perspective=0.0007, fliplr=0.5)
    for i, x in enumerate(d):
        x["perspective"] = i % 3 == 0
    return d


def test_training_batch_over_several_chunks_equals_the_oracle():
    import yfv2_engine as eng
    N, H, W = 256, 352, 352
    rs = np.random.RandomState(5)
    x = torch.from_numpy(rs.randint(0, 256, (N, 3, H, W)).astype(np.uint8)).cuda()
    d = mixed_draws(N, H, W, 6)
    assert 0 < sum(v["mosaic"] for v in d) < N and any(v["perspective"] for v in d) and any(v["flip"] for v in d)
    got = eng.augment_geometric(x, d).cpu().numpy()
    assert np.array_equal(got, go.augment_planar(x.cpu().numpy(), d))


@pytest.mark.parametrize("H,W", [(37, 53), (1, 7), (19, 1), (65, 129)])
def test_odd_sizes_and_unaligned_bases(H, W):
    import yfv2_engine as eng
    N = 5
    rs = np.random.RandomState(H * W)
    host = rs.randint(0, 256, (N, 3, H, W)).astype(np.uint8)
    buf = torch.empty(N * 3 * H * W + 3, dtype=torch.uint8, device="cuda")
    x = buf[1:1 + host.size].view(N, 3, H, W)
    x.copy_(torch.from_numpy(host))
    obuf = torch.full((N * 3 * H * W + 5,), 7, dtype=torch.uint8, device="cuda")
    out = obuf[3:3 + host.size].view(N, 3, H, W)
    d = mixed_draws(N, H, W, 7, mosaic=0)
    for v in d:
        v["src"] = [(v["src"][0] + 2) % N] * 4
    assert eng.augment_geometric(x, d, out=out) is out
    assert np.array_equal(out.cpu().numpy(), go.augment_planar(host, d))
    assert (obuf[:3] == 7).all() and (obuf[3 + host.size:] == 7).all()                # nothing written outside out


def test_flip_only_is_torch_flip_and_identity_is_the_input():
    import yfv2_engine as eng
    rs = np.random.RandomState(8)
    x = torch.from_numpy(rs.randint(0, 256, (6, 3, 40, 72)).astype(np.uint8)).cuda()
    ident = [dict(M=np.eye(3), perspective=False, mosaic=False, src=[i] * 4, flip=False) for i in range(6)]
    assert torch.equal(eng.augment_geometric(x, ident), x)
    flip = [dict(v, flip=True) for v in ident]
    assert torch.equal(eng.augment_geometric(x, flip), torch.flip(x, [3]))
    persp = [dict(v, perspective=True) for v in flip]
    assert torch.equal(eng.augment_geometric(x, persp), torch.flip(x, [3]))


def test_overlap_is_refused():
    import yfv2_engine as eng
    x = torch.zeros((2, 3, 8, 8), dtype=torch.uint8, device="cuda")
    d = [dict(M=np.eye(3), perspective=False, mosaic=False, src=[i] * 4, flip=False) for i in range(2)]
    with pytest.raises(eng.Yfv2Error, match="overlap"):
        eng.augment_geometric(x, d, out=x)


def rect_batch(N, H, W, seed):
    """Flat black images with up to three solid rectangles each, every rectangle in a colour of its own (B = 10 k, G = 250 - 10 k,
    R = 200 for rectangle k), and their targets (class k)."""
    rs = np.random.RandomState(seed)
    imgs = np.zeros((N, 3, H, W), np.uint8)
    rows, k = [], 1
    for n in range(N):
        taken = np.zeros((H, W), bool)
        for _ in range(3):
            w, h = rs.randint(12, W // 2), rs.randint(12, H // 2)
            x0, y0 = rs.randint(-w // 3, W - 2 * w // 3), rs.randint(-h // 3, H - 2 * h // 3)
            xa, ya, xb, yb = max(x0, 0), max(y0, 0), min(x0 + w, W), min(y0 + h, H)
            if taken[max(ya - 3, 0):yb + 3, max(xa - 3, 0):xb + 3].any():
                continue
            taken[ya:yb, xa:xb] = True
            imgs[n, :, ya:yb, xa:xb] = np.array([10 * k, 250 - 10 * k, 200], np.uint8)[:, None, None]
            rows.append([n, k, (xa + xb) / 2 / W, (ya + yb) / 2 / H, (xb - xa) / W, (yb - ya) / H])
            k += 1
    return imgs, np.array(rows, np.float32)


def test_labels_move_with_the_pixels():
    """Each output label bounds its rectangle's pixels within 2 px (affine, no rotation or shear), through mosaics, clipping at
    every border and flips."""
    import utils.device_aug as da
    N, H, W = 8, 96, 128
    imgs, t = rect_batch(N, H, W, 9)
    assert len(t) >= 12
    x = torch.from_numpy(imgs).cuda()
    checked = 0
    for seed in range(4):
        out, tt = da.geometric_batch(x, torch.from_numpy(t), random.Random(seed), mosaic=0.6, degrees=0, shear=0, translate=0.2,
                                     scale=0.4, perspective=0, fliplr=0.5)
        out = out.cpu().numpy()
        for row in tt.numpy():
            n, k = int(row[0]), int(row[1])
            x1, x2 = (row[2] - row[4] / 2) * W, (row[2] + row[4] / 2) * W
            y1, y2 = (row[3] - row[5] / 2) * H, (row[3] + row[5] / 2) * H
            if x2 - x1 < 4 or y2 - y1 < 4:
                continue
            # the label's window, 3 px wider: a mosaic may show the same image, and so the same rectangle, in two tiles
            wx, wy = max(int(x1) - 3, 0), max(int(y1) - 3, 0)
            o = out[n, :, wy:int(y2) + 4, wx:int(x2) + 4].astype(int)
            m = (np.abs(o[0] - 10 * k) <= 2) & (np.abs(o[1] - (250 - 10 * k)) <= 2) & (np.abs(o[2] - 200) <= 2)
            ys, xs = np.nonzero(m)
            assert len(xs), (seed, n, k)
            ext = np.array([xs.min() + wx, ys.min() + wy, xs.max() + 1 + wx, ys.max() + 1 + wy])
            assert np.abs(ext - [x1, y1, x2, y2]).max() <= 2, (seed, n, k, ext, (x1, y1, x2, y2))
            checked += 1
    assert checked >= 30


def test_geometric_batch_then_img_aug_into_a_second_buffer():
    import utils.device_aug as da
    imgs, t = rect_batch(4, 64, 64, 10)
    x = torch.from_numpy(imgs).cuda()
    buf = torch.empty_like(x)
    out, tt = da.geometric_batch(x, torch.from_numpy(t).pin_memory(), random.Random(1), out=buf)
    assert out is buf and tt.is_pinned() and tt.dtype == torch.float32
    d = da.draw_geometric(4, 64, 64, random.Random(1))
    assert np.array_equal(buf.cpu().numpy(), go.augment_planar(imgs, d))
    assert torch.equal(tt, da.geometric_targets(torch.from_numpy(t), d, 64, 64))


def _data(tmp_path):
    names = tmp_path / "coco.names"
    names.write_text("\n".join("c%d" % i for i in range(80)) + "\n")
    data = tmp_path / "coco.data"
    data.write_text("[name]\nmodel_name=coco\n\n[train-configure]\nepochs=1\nsteps=150,250\nbatch_size=64\nsubdivisions=1\n"
                    "learning_rate=0.001\n\n[model-configure]\npre_weights=None\nclasses=80\nwidth=352\nheight=352\nanchor_num=3\n"
                    "anchors=12.64,19.39, 37.88,51.48, 55.71,138.31, 126.91,78.23, 131.57,214.55, 279.92,258.87\n\n"
                    "[data-configure]\ntrain=/nonexistent/train.txt\nval=/nonexistent/val.txt\nnames=%s\n" % names)
    return str(data)


def test_trainer_runs_with_geometric_augmentation(tmp_path, monkeypatch):
    import train_dist
    import utils.device_aug
    import utils.loss
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    data = _data(tmp_path)
    real_loss, real_geom = utils.loss.compute_loss, utils.device_aug.geometric_batch
    losses, targets = [], []

    def loss(*a, **kw):
        r = real_loss(*a, **kw)
        losses[-1].append([float(v.detach()) for v in r[:4]])
        return r

    def geom(imgs, t, *a, **kw):
        r = real_geom(imgs, t, *a, **kw)
        targets[-1].append(r[1].clone())
        return r
    monkeypatch.setattr(utils.loss, "compute_loss", loss)
    monkeypatch.setattr(utils.device_aug, "geometric_batch", geom)
    for _ in range(2):
        losses.append([])
        targets.append([])
        random.seed(12)
        np.random.seed(12)
        train_dist.main(["--data", data, "--synthetic", "64", "--device-aug", "--device-aug-geom", "--max-iters", "3", "--epochs", "3"])
    assert len(losses[0]) == 3 and np.isfinite(losses[0]).all()
    np.testing.assert_allclose(losses[1], losses[0], rtol=1e-5)
    assert len(targets[0]) == 3 and all(torch.equal(a, b) for a, b in zip(targets[0], targets[1]))
    losses.append([])
    targets.append([])
    train_dist.main(["--data", data, "--synthetic", "64", "--device-aug", "--device-aug-geom", "mosaic=0,fliplr=1,degrees=5",
                     "--max-iters", "1"])
    assert len(targets[-1]) == 1 and np.isfinite(losses[-1]).all()


def test_trainer_without_the_flag_never_augments_geometrically(tmp_path, monkeypatch):
    import train_dist
    import utils.device_aug
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)

    def fail(*a, **kw):
        raise AssertionError("geometric augmentation without --device-aug-geom")
    monkeypatch.setattr(utils.device_aug, "geometric_batch", fail)
    monkeypatch.setattr(utils.device_aug, "draw_geometric", fail)
    net = train_dist.main(["--data", _data(tmp_path), "--synthetic", "64", "--device-aug", "--max-iters", "2"])
    assert all(torch.isfinite(p).all() for p in net.parameters())

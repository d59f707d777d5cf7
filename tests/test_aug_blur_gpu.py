"""yfv2_aug_batch_blur (contrast -> motion_blur -> random_resize -> augment_hsv) against cv2 / reference goldens
(tests/golden/aug_blur_cases.npz) and the oracles (tests/aug_blur_oracle.py, tests/aug_hsv_oracle.py): bit-exact bytes."""
import hashlib
import os
import random

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import yfv2_engine as eng
import aug_blur_cases as bc
import aug_blur_oracle as bo
import aug_hsv_oracle as ho
from oracle import aug as oaug

pytestmark = pytest.mark.gpu


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest()


@pytest.fixture(scope="module")
def g(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "aug_blur_cases.npz")))


def planar(imgs):                     # [h, w, 3] images -> CUDA [n, 3, h, w]
    return torch.from_numpy(np.stack([np.ascontiguousarray(i.transpose(2, 0, 1)) for i in imgs])).cuda()


def packed(t):                        # CUDA [3, h, w] -> [h, w, 3]
    return t.cpu().numpy().transpose(1, 2, 0)


def filter_cases():
    cases = [(n, bc.image(*spec), d, a) for n, spec, d, a in bc.FILTER_CASES]
    return cases + [("constant", bc.constant_image(), 3, 27.0), ("striped", bc.striped_image(), 2, 0.0)]


@pytest.mark.parametrize("name,img,d,a", filter_cases(), ids=[c[0] for c in filter_cases()])
def test_motion_blur_golden(g, name, img, d, a):
    got = eng.augment_batch(planar([img]), blur=[(d, a)])
    assert sha(packed(got[0])) == g["norm_%s_sha256" % name].tobytes()


@pytest.mark.parametrize("s", bc.BLUR_SEEDS)
def test_seeded_motion_blur_golden(g, s):
    dr = g["blur_%d_draws" % s]
    blur = [(int(d), a) if first == 1 else None for first, d, a in dr]
    got = eng.augment_batch(planar(bc.seeded_batch(s)), blur=blur)
    for i in range(bc.SEEDED_N):
        assert sha(packed(got[i])) == g["blur_%d_%d_sha256" % (s, i)].tobytes(), (s, i)


@pytest.mark.parametrize("s", bc.CHAIN_SEEDS)
def test_img_aug_batch_seeded_equals_the_reference_chain(g, s):
    import utils.device_aug as da
    batch = planar(bc.seeded_batch(s))
    kw = dict(random_resize=True, augment_hsv=True, motion_blur=True)
    got = da.img_aug_batch(batch, random.Random(s), np_rng=np.random.RandomState(s), **kw)
    for i in range(bc.SEEDED_N):
        assert sha(packed(got[i])) == g["chain_%d_%d_sha256" % (s, i)].tobytes(), (s, i)
    before = batch.clone()
    res = da.img_aug_batch(batch, random.Random(s), out=batch, np_rng=np.random.RandomState(s), **kw)
    assert res is batch and torch.equal(batch, got) and not torch.equal(before, got)


def draws(n, H, W, seed, every=3):
    """Per-image parameters; image i draws no blur when i % every == every - 1 (every 0: all blurred)."""
    rs = np.random.RandomState(seed)
    a, b = rs.uniform(0.25, 1.75, n), rs.uniform(0.25, 1.75, n)
    rw = np.maximum((W * rs.uniform(0.8, 1, n)).astype(int), 1)
    rh = np.maximum((H * rs.uniform(0.8, 1, n)).astype(int), 1)
    r = rs.uniform(-1, 1, (n, 3)) * list(ho.HSV_GAINS) + 1
    blur = [(int(rs.randint(2, 4)), float(rs.uniform(-360, 360))) for _ in range(n)]
    if every:
        blur = [None if i % every == every - 1 else blur[i] for i in range(n)]
    return a, b, rw, rh, r, blur


def oracle(src, flags, a, b, rw, rh, r, blur, memo=None):
    """One packed image through the steps flags selects (1 contrast, 2 resize, 4 HSV, 8 blur), in img_aug's order.  memo: a
    dict that keeps the image after contrast and blur between calls on the same src."""
    key = flags & 9
    if memo is None or key not in memo:
        x = oaug.contrast_and_brightness(src, a, b) if flags & 1 else src
        if flags & 8 and blur is not None:
            x = bo.motion_blur(x, *blur)
        if memo is not None:
            memo[key] = x
    x = memo[key] if memo is not None else x
    if flags & 2:
        x = ho.random_resize(x, rw, rh)
    if flags & 4:
        x = ho.augment_hsv(x, r)
    return x


@pytest.mark.parametrize("N,H,W,offset,every", [(64, 352, 352, 0, 0), (6, 37, 53, 0, 3), (4, 33, 47, 1, 2), (3, 16, 1, 3, 3),
                                                (2, 1, 45, 0, 0), (3, 2, 2, 0, 3)])
def test_all_flag_combinations_equal_the_oracle(N, H, W, offset, every):
    rs = np.random.RandomState(N * 1000 + H)
    x = rs.randint(0, 256, (N, 3, H, W)).astype(np.uint8)
    a, b, rw, rh, r, blur = draws(N, H, W, H + W, every)
    luts = eng.hsv_luts(r)
    base = torch.empty(N * 3 * H * W + 16, dtype=torch.uint8, device="cuda")
    img = base[offset:offset + x.size].view(N, 3, H, W)             # a base that is not 16-byte aligned when offset > 0
    img.copy_(torch.from_numpy(x))
    memos = [{} for _ in range(N)]
    for flags in range(16):
        got = eng.augment_batch(img, a if flags & 1 else None, b if flags & 1 else None, rw if flags & 2 else None,
                                rh if flags & 2 else None, luts if flags & 4 else None,
                                blur=blur if flags & 8 else [None] * N).cpu().numpy()
        for n in range(N):
            want = oracle(x[n].transpose(1, 2, 0), flags, a[n], b[n], rw[n], rh[n], r[n], blur[n], memos[n])
            assert np.array_equal(got[n].transpose(1, 2, 0), want), (flags, n)


def test_blur_entry_without_blurred_images_equals_aug_batch():
    rs = np.random.RandomState(5)
    x = torch.from_numpy(rs.randint(0, 256, (9, 3, 64, 80)).astype(np.uint8)).cuda()
    a, b, rw, rh, r, _ = draws(9, 64, 80, 1)
    luts = eng.hsv_luts(r)
    for args in ((a, b, None, None, None), (a, b, rw, rh, luts), (None, None, None, None, luts)):
        assert torch.equal(eng.augment_batch(x, *args, blur=[None] * 9), eng.augment_batch(x, *args))


@pytest.mark.parametrize("resize", [False, True])
def test_mixed_batch_across_the_chunk_boundary(resize):
    N, H, W = 130, 48, 72
    rs = np.random.RandomState(130 + resize)
    x = rs.randint(0, 256, (N, 3, H, W)).astype(np.uint8)
    a, b, rw, rh, r, blur = draws(N, H, W, 7, 4)
    blur[127], blur[128], blur[129] = (3, 21.5), None, (2, -100.25)
    luts = eng.hsv_luts(r)
    got = eng.augment_batch(torch.from_numpy(x).cuda(), a, b, rw if resize else None, rh if resize else None, luts,
                            blur=blur).cpu().numpy()
    flags = 1 | 4 | 8 | (2 if resize else 0)
    for n in range(N):
        want = oracle(x[n].transpose(1, 2, 0), flags, a[n], b[n], rw[n], rh[n], r[n], blur[n])
        assert np.array_equal(got[n].transpose(1, 2, 0), want), n


def test_constant_images_become_zero():
    imgs = [bc.constant_image(24, 40, 77), bc.striped_image(24, 40), bc.constant_image(24, 40, 0), bc.constant_image(24, 40, 255)]
    x = planar(imgs)
    got = eng.augment_batch(x, blur=[(3, 27.0), (2, 0.0), (2, 45.0), None])
    assert not got[:3].any() and torch.equal(got[3], x[3])
    # contrast that saturates every byte makes the image constant before the blur
    sat = planar([np.full((24, 40, 3), 200, np.uint8)])
    assert not eng.augment_batch(sat, [1.75], [1.75], blur=[(3, 60.0)]).any()


@pytest.mark.parametrize("H,W", [(352, 352), (37, 53)])
def test_in_place_without_resize(H, W):
    rs = np.random.RandomState(H)
    x = rs.randint(0, 256, (6, 3, H, W)).astype(np.uint8)
    a, b, _, _, r, blur = draws(6, H, W, 3)
    luts = eng.hsv_luts(r)
    for ab, lt in (((a, b), None), ((None, None), luts), ((a, b), luts)):
        want = eng.augment_batch(torch.from_numpy(x).cuda(), *ab, luts=lt, blur=blur)
        d = torch.from_numpy(x).cuda()
        assert eng.augment_batch(d, *ab, luts=lt, out=d, blur=blur) is d and torch.equal(d, want)


def test_trainer_runs_with_all_device_augmentations(tmp_path, monkeypatch):
    import train_dist
    names = tmp_path / "coco.names"
    names.write_text("\n".join("c%d" % i for i in range(80)) + "\n")
    data = tmp_path / "coco.data"
    data.write_text("[name]\nmodel_name=coco\n\n[train-configure]\nepochs=1\nsteps=150,250\nbatch_size=64\nsubdivisions=1\n"
                    "learning_rate=0.001\n\n[model-configure]\npre_weights=None\nclasses=80\nwidth=352\nheight=352\nanchor_num=3\n"
                    "anchors=12.64,19.39, 37.88,51.48, 55.71,138.31, 126.91,78.23, 131.57,214.55, 279.92,258.87\n\n"
                    "[data-configure]\ntrain=/nonexistent/train.txt\nval=/nonexistent/val.txt\nnames=%s\n" % names)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    net = train_dist.main(["--data", str(data), "--synthetic", "512", "--max-iters", "20", "--device-aug", "--device-aug-resize",
                           "--device-aug-hsv", "--device-aug-blur"])
    assert all(torch.isfinite(p).all() for p in net.parameters())
    with pytest.raises(SystemExit):
        train_dist.main(["--data", str(data), "--synthetic", "16", "--device-aug-blur"])

"""yfv2_aug_batch (contrast -> random_resize -> augment_hsv in one pass) and the HSV conversion hooks against cv2 / reference
goldens (tests/golden/aug_hsv_cases.npz) and the oracle (tests/aug_hsv_oracle.py): bit-exact bytes."""
import hashlib
import os
import random

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import yfv2_engine as eng
import aug_hsv_cases as hc
import aug_hsv_oracle as ho
from oracle import aug as oaug

pytestmark = pytest.mark.gpu


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest()


@pytest.fixture(scope="module")
def g(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "aug_hsv_cases.npz")))


def planar(img):                      # [h, w, 3] -> CUDA [1, 3, h, w]
    return torch.from_numpy(np.ascontiguousarray(img.transpose(2, 0, 1)))[None].cuda()


def packed(t):                        # CUDA [3, h, w] -> [h, w, 3]
    return t.cpu().numpy().transpose(1, 2, 0)


def test_debug_hooks_over_all_byte_triples_match_cv2(g):
    cube = torch.from_numpy(ho.all_triples()).cuda()
    hsv = eng.debug_bgr2hsv(cube)
    assert sha(hsv.cpu().numpy()) == g["bgr2hsv_sha256"].tobytes()
    assert sha(eng.debug_hsv2bgr(cube).cpu().numpy()) == g["hsv2bgr_sha256"].tobytes()
    assert sha(eng.debug_hsv2bgr(hsv).cpu().numpy()) == g["roundtrip_sha256"].tobytes()
    assert sha(eng.debug_hsv2bgr(cube.reshape(-1, 1, 3)).cpu().numpy()) == g["hsv2bgr_col_sha256"].tobytes()
    w53 = cube[:, :4081].contiguous().reshape(-1, 53, 3)
    assert sha(eng.debug_hsv2bgr(w53).cpu().numpy()) == g["hsv2bgr_w53_sha256"].tobytes()


@pytest.mark.parametrize("name,img_spec,u", hc.HSV_CASES, ids=[c[0] for c in hc.HSV_CASES])
def test_augment_hsv_golden(g, name, img_spec, u):
    got = eng.augment_batch(planar(hc.image(*img_spec)), luts=g["hsv_%s_luts" % name][None])
    assert sha(packed(got[0])) == g["hsv_%s_sha256" % name].tobytes()


@pytest.mark.parametrize("name,img_spec,size", hc.RESIZE_CASES, ids=[c[0] for c in hc.RESIZE_CASES])
def test_random_resize_golden(g, name, img_spec, size):
    got = eng.augment_batch(planar(hc.image(*img_spec)), rw=[size[0]], rh=[size[1]])
    assert sha(packed(got[0])) == g["rr_%s_sha256" % name].tobytes()


def test_random_resize_seeded_golden(g):
    for s in hc.RESIZE_SEEDS:
        rw, rh = int(g["rr_seed%d_rw" % s]), int(g["rr_seed%d_rh" % s])
        got = eng.augment_batch(planar(hc.image(40 + s, 352, 352)), rw=[rw], rh=[rh])
        assert sha(packed(got[0])) == g["rr_seed%d_sha256" % s].tobytes(), s


@pytest.mark.parametrize("s", hc.CHAIN_SEEDS)
def test_img_aug_batch_seeded_equals_the_reference_chain(g, s):
    import utils.device_aug as da
    batch = torch.cat([planar(img) for img in hc.chain_batch(s)])
    got = da.img_aug_batch(batch, random.Random(s), random_resize=True, augment_hsv=True, np_rng=np.random.RandomState(s))
    for i in range(hc.CHAIN_N):
        assert sha(packed(got[i])) == g["chain_%d_%d_sha256" % (s, i)].tobytes(), (s, i)
    before = batch.clone()                                         # in place goes through a scratch buffer
    res = da.img_aug_batch(batch, random.Random(s), out=batch, random_resize=True, augment_hsv=True,
                           np_rng=np.random.RandomState(s))
    assert res is batch and torch.equal(batch, got) and not torch.equal(before, got)


def draws(n, H, W, seed):
    rs = np.random.RandomState(seed)
    a, b = rs.uniform(0.25, 1.75, n), rs.uniform(0.25, 1.75, n)
    rw = np.maximum((W * rs.uniform(0.8, 1, n)).astype(int), 1)      # int(1 * u) = 0 would be refused (cv2 refuses it too)
    rh = np.maximum((H * rs.uniform(0.8, 1, n)).astype(int), 1)
    rw[0], rh[0] = W, H                                            # the identity size
    if n > 1:
        rw[1], rh[1] = 1, 1
    r = rs.uniform(-1, 1, (n, 3)) * list(ho.HSV_GAINS) + 1
    return a, b, rw, rh, r


@pytest.mark.parametrize("N,H,W,offset", [(64, 352, 352, 0), (5, 37, 53, 0), (4, 33, 47, 1), (3, 16, 1, 3), (2, 1, 45, 0)])
def test_all_flag_combinations_equal_the_oracle(N, H, W, offset):
    rs = np.random.RandomState(N * 1000 + H)
    x = rs.randint(0, 256, (N, 3, H, W)).astype(np.uint8)
    a, b, rw, rh, r = draws(N, H, W, H + W)
    luts = eng.hsv_luts(r)
    base = torch.empty(N * 3 * H * W + 16, dtype=torch.uint8, device="cuda")
    img = base[offset:offset + x.size].view(N, 3, H, W)             # a base that is not 16-byte aligned when offset > 0
    img.copy_(torch.from_numpy(x))
    for flags in range(8):
        got = eng.augment_batch(img, a if flags & 1 else None, b if flags & 1 else None, rw if flags & 2 else None,
                                rh if flags & 2 else None, luts if flags & 4 else None).cpu().numpy()
        for n in range(N):
            src = x[n].transpose(1, 2, 0)
            want = ho.img_aug(src, a[n], b[n]) if flags & 1 else src
            if flags & 2:
                want = ho.random_resize(want, rw[n], rh[n])
            if flags & 4:
                want = ho.augment_hsv(want, r[n])
            assert np.array_equal(got[n].transpose(1, 2, 0), want), (flags, n)


def test_contrast_only_equals_the_existing_kernel():
    rs = np.random.RandomState(9)
    x = torch.from_numpy(rs.randint(0, 256, (16, 3, 352, 352)).astype(np.uint8)).cuda()
    a, b = rs.uniform(0.25, 1.75, 16), rs.uniform(0.25, 1.75, 16)
    assert torch.equal(eng.augment_batch(x, a, b), eng.contrast_and_brightness(x, a, b))


@pytest.mark.parametrize("H,W", [(352, 352), (37, 53)])
def test_in_place_without_resize(H, W):
    rs = np.random.RandomState(H)
    x = rs.randint(0, 256, (6, 3, H, W)).astype(np.uint8)
    a, b, _, _, r = draws(6, H, W, 3)
    luts = eng.hsv_luts(r)
    for ab, lt in (((a, b), None), ((None, None), luts), ((a, b), luts)):
        want = eng.augment_batch(torch.from_numpy(x).cuda(), *ab, luts=lt)
        d = torch.from_numpy(x).cuda()
        assert eng.augment_batch(d, *ab, luts=lt, out=d) is d and torch.equal(d, want)


def test_img_aug_batch_defaults_are_unchanged():
    import utils.device_aug as da
    rs = np.random.RandomState(4)
    x = torch.from_numpy(rs.randint(0, 256, (8, 3, 64, 80)).astype(np.uint8)).cuda()
    rng = random.Random(3)
    got = da.img_aug_batch(x, random.Random(3))
    ab = [(rng.uniform(0.25, 1.75), rng.uniform(0.25, 1.75)) for _ in range(8)]
    want = np.stack([oaug.contrast_and_brightness(x[i].cpu().numpy(), *ab[i]) for i in range(8)])
    assert np.array_equal(got.cpu().numpy(), want)


def test_trainer_runs_with_device_resize_and_hsv(tmp_path, monkeypatch):
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
                           "--device-aug-hsv"])
    assert all(torch.isfinite(p).all() for p in net.parameters())
    with pytest.raises(SystemExit):
        train_dist.main(["--data", str(data), "--synthetic", "16", "--device-aug-hsv"])

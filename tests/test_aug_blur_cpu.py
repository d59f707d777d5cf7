"""motion_blur restatement (tests/aug_blur_oracle.py) and yfv2_engine.motion_blur_taps against the real cv2 and the reference
(tests/golden/aug_blur_cases.npz), img_aug's draw order with motion_blur, and every refusal of yfv2_aug_batch_blur before
anything is launched."""
import ctypes
import hashlib
import math
import os
import random

import numpy as np
import pytest

import yfv2  # noqa: F401
import aug_blur_cases as bc
import aug_blur_oracle as bo
import aug_hsv_oracle as ho


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest()


@pytest.fixture(scope="module")
def g(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "aug_blur_cases.npz")))


@pytest.mark.parametrize("d", [2, 3])
def test_taps_sweep_match_cv2(g, d):
    import yfv2_engine as eng
    assert sha(np.stack([bo.taps(d, a) for a in bc.SWEEP])) == g["sweep_d%d_sha256" % d].tobytes()
    assert sha(np.stack([eng.motion_blur_taps(d, a) for a in bc.SWEEP])) == g["sweep_d%d_sha256" % d].tobytes()
    for i, a in enumerate(bc.FULL_ANGLES):
        want = g["taps_d%d_%d" % (d, i)]
        assert want.dtype == np.float32 and want.shape == (d, d)
        assert np.array_equal(bo.taps(d, a), want) and np.array_equal(eng.motion_blur_taps(d, a), want), a


@pytest.mark.parametrize("d", [2, 3])
def test_taps_at_special_angles_and_rounding_edges(g, d):
    import yfv2_engine as eng
    for a, want in zip(bc.SPECIAL_ANGLES, g["special_d%d_taps" % d]):
        assert np.array_equal(bo.taps(d, a), want) and np.array_equal(eng.motion_blur_taps(d, a), want), a
    for which, name in ((0, "edge1024"), (1, "edge32")):
        pairs = g["%s_d%d" % (name, d)]
        assert len(pairs) >= 6
        for (a0, a1), want in zip(pairs, g["%s_d%d_taps" % (name, d)]):
            assert np.nextafter(a0, a1) == a1                                # adjacent doubles ...
            assert bc.fixed_terms(d, a0)[which] != bc.fixed_terms(d, a1)[which]   # ... on either side of the edge
            for a, w in zip((a0, a1), want):
                assert np.array_equal(bo.taps(d, a), w) and np.array_equal(eng.motion_blur_taps(d, a), w), (name, a)


def test_special_angles_are_the_expected_kernels(g):
    for d in (2, 3):
        k0 = g["special_d%d_taps" % d][0]                                   # angle 0: the diagonal over degree
        assert np.array_equal(k0, (np.eye(d) / d).astype(np.float32))


def filter_cases():
    cases = [(n, bc.image(*spec), d, a) for n, spec, d, a in bc.FILTER_CASES]
    return cases + [("constant", bc.constant_image(), 3, 27.0), ("striped", bc.striped_image(), 2, 0.0)]


@pytest.mark.parametrize("name,img,d,a", filter_cases(), ids=[c[0] for c in filter_cases()])
def test_filter2d_and_normalize_match_cv2(g, name, img, d, a):
    f = bo.filter2d(img, bo.taps(d, a))
    assert sha(f) == g["filt_%s_sha256" % name].tobytes()
    assert sha(bo.normalize(f)) == g["norm_%s_sha256" % name].tobytes()
    if name in ("constant", "striped"):
        assert f.min() == f.max() and not bo.normalize(f).any()


def test_normalize_map_edges():
    assert not bo.normalize_map(77, 77).any()                               # constant: all zeros
    m = bo.normalize_map(3, 250)
    assert m[3] == 0 and m[250] == 255 and np.all(np.diff(m[3:251].astype(int)) >= 0)
    assert np.array_equal(bo.normalize_map(0, 255), np.arange(256))


@pytest.mark.parametrize("s", bc.BLUR_SEEDS)
def test_seeded_motion_blur_equals_the_reference(g, s):
    draws = g["blur_%d_draws" % s]
    assert set(draws[:, 0]) == {1.0, 2.0}                                   # both branches drawn
    for i, img in enumerate(bc.seeded_batch(s)):
        first, degree, angle = draws[i]
        got = bo.motion_blur(img, int(degree), angle) if first == 1 else img
        assert sha(got) == g["blur_%d_%d_sha256" % (s, i)].tobytes(), (s, i)


@pytest.mark.parametrize("s", bc.CHAIN_SEEDS)
def test_chain_equals_the_reference(g, s):
    from oracle import aug as oaug
    for i, img in enumerate(bc.seeded_batch(s)):
        x = oaug.contrast_and_brightness(img, g["chain_%d_alpha" % s][i], g["chain_%d_beta" % s][i])
        d = int(g["chain_%d_degree" % s][i])
        if d:
            x = bo.motion_blur(x, d, g["chain_%d_angle" % s][i])
        x = ho.augment_hsv(ho.random_resize(x, int(g["chain_%d_rw" % s][i]), int(g["chain_%d_rh" % s][i])), g["chain_%d_r" % s][i])
        assert sha(x) == g["chain_%d_%d_sha256" % (s, i)].tobytes(), (s, i)


class Recorder:
    """A random.Random whose uniform / randint calls are logged as (kind, value) like the golden's chain_<seed>_calls."""
    def __init__(self, seed, np_seed):
        self.r, self.np, self.calls = random.Random(seed), np.random.RandomState(np_seed), []

    def uniform(self, lo, hi):
        v = self.r.uniform(lo, hi)
        self.calls.append((0, v))
        return v

    def randint(self, lo, hi):
        v = self.r.randint(lo, hi)
        self.calls.append((1, v))
        return v


class NpRecorder:
    def __init__(self, rec):
        self.rec = rec

    def uniform(self, lo, hi, n):
        v = self.rec.np.uniform(lo, hi, n)
        self.rec.calls.extend((2, x) for x in v)
        return v


@pytest.mark.parametrize("s", bc.CHAIN_SEEDS)
def test_draw_order_equals_the_reference(g, s):
    import utils.device_aug as da
    rec = Recorder(s, s)
    alpha, beta, blur, rw, rh, gains = da.draw(bc.SEEDED_N, 352, 352, rec, NpRecorder(rec), motion_blur=True, random_resize=True,
                                               augment_hsv=True)
    want = g["chain_%d_calls" % s]
    assert np.array_equal(np.array(rec.calls, np.float64), want)
    assert [b[0] if b else 0 for b in blur] == g["chain_%d_degree" % s].tolist()
    assert rw == g["chain_%d_rw" % s].tolist() and np.array_equal(np.stack(gains), g["chain_%d_r" % s])


def test_chain_seeds_cover_both_branches(g):
    degrees = np.concatenate([g["chain_%d_degree" % s] for s in bc.CHAIN_SEEDS])
    assert set(degrees.tolist()) == {0, 2, 3}


def test_draws_without_motion_blur_are_unchanged():
    import utils.device_aug as da
    for kw in (dict(), dict(random_resize=True), dict(augment_hsv=True), dict(random_resize=True, augment_hsv=True)):
        a, b, blur, rw, rh, gains = da.draw(5, 40, 30, random.Random(1), np.random.RandomState(1), **kw)
        r = random.Random(1)
        nr = np.random.RandomState(1)
        for i in range(5):
            assert (a[i], b[i]) == (r.uniform(0.25, 1.75), r.uniform(0.25, 1.75))
            if kw.get("random_resize"):
                assert (rw[i], rh[i]) == (int(30 * r.uniform(0.8, 1)), int(40 * r.uniform(0.8, 1)))
        if kw.get("augment_hsv"):
            assert np.array_equal(np.stack(gains), nr.uniform(-1, 1, (5, 3)) * [0.0138, 0.678, 0.36] + 1)
        assert blur == []


def test_motion_blur_taps_refuses_other_degrees():
    import yfv2_engine as eng
    for d in (0, 1, 4):
        with pytest.raises(ValueError):
            eng.motion_blur_taps(d, 10.0)


# ---- yfv2_aug_batch_blur refusals: checked on the host before any launch, so this runs without a GPU ---------------------------
N_, H_, W_ = 2, 8, 8
IMG_BYTES = N_ * 3 * H_ * W_


def ws_bytes(N=N_, H=H_, W=W_):
    import yfv2_engine as eng
    nb = ctypes.c_size_t()
    assert eng.lib().yfv2_aug_blur_workspace_bytes(N, H, W, ctypes.byref(nb)) == 0
    return nb.value


DEFAULT_BLUR = ((3, (0.1,) * 9), (0, ()))


IMG, OUT, WS = 1 << 24, 1 << 25, 1 << 26


def call(img=IMG, out=OUT, N=N_, H=H_, W=W_, params=((1.0, 0.0, 8, 8), (1.0, 0.0, 8, 8)), luts=1, blur=DEFAULT_BLUR, flags=15,
         ws=WS, nws=None):
    import yfv2_engine as eng
    L = eng.lib()
    arr = (eng.AugParams * max(len(params or ()), 1))(*[eng.AugParams(*p) for p in (params or ())])
    barr = None
    if blur is not None:
        barr = (eng.AugBlur * len(blur))()
        for i, (k, t) in enumerate(blur):
            barr[i].ksize = k
            for j, v in enumerate(t):
                barr[i].taps[j] = v
    p = lambda v: ctypes.c_void_p(v) if v else None                        # never dereferenced: the checks come first
    rc = L.yfv2_aug_batch_blur(p(img), p(out), N, H, W, arr if params is not None else None, p(luts), barr, flags, p(ws),
                               ws_bytes() if nws is None else nws, None)
    return rc, L.yfv2_last_error().decode()


@pytest.mark.parametrize("kw,msg", [
    (dict(img=0), "null img"), (dict(params=None), "params"), (dict(N=0), "N <= 0"), (dict(H=0), "outside"),
    (dict(W=40000), "outside"), (dict(flags=16), "unknown flags"), (dict(flags=-1), "unknown flags"), (dict(luts=0), "needs luts"),
    (dict(blur=None), "needs blur descriptors"), (dict(ws=0), "needs a workspace"), (dict(nws=1), "needs a workspace"),
    (dict(blur=((1, (0.5,)), (0, ()))), "image 0: blur ksize 1"), (dict(blur=((3, (0.1,) * 9), (4, ()))), "image 1: blur ksize 4"),
    (dict(blur=((3, (0.1,) * 9), (-1, ()))), "image 1: blur ksize -1"),
    (dict(blur=((2, (0.5, math.nan, 0.0, 0.5)), (0, ()))), "image 0: blur tap 1 is not finite"),
    (dict(blur=((3, (0.1,) * 8 + (math.inf,)), (0, ()))), "image 0: blur tap 8 is not finite"),
    (dict(blur=((0, ()), (2, (0.5, 0.0, -math.inf, 0.5)))), "image 1: blur tap 2 is not finite"),
    (dict(out=IMG), "img and out overlap"), (dict(out=IMG + 1, flags=9), "img and out overlap"),
    (dict(ws=IMG + IMG_BYTES - 1), "workspace overlaps"), (dict(ws=OUT + 5), "workspace overlaps"),
    (dict(ws=IMG - ws_bytes() + 1, flags=9), "workspace overlaps"), (dict(ws=IMG, out=IMG, flags=9), "workspace overlaps"),
    (dict(params=((1.0, 0.0, 0, 8), (1.0, 0.0, 8, 8))), "image 0: random_resize size 0x8"),
])
def test_aug_batch_blur_refusals_before_any_launch(kw, msg):
    rc, err = call(**kw)
    assert rc == -1 and msg in err, (rc, err)


def test_aug_batch_blur_refusals_accept_the_edges_without_a_device():
    """The edges that pass the checks reach the first CUDA call, which fails with YFV2_ECUDA here for want of a device."""
    torch = pytest.importorskip("torch")
    if torch.cuda.is_available():
        pytest.skip("the launch would read the fake pointers")
    for kw in (dict(), dict(out=IMG, flags=9), dict(ws=IMG + IMG_BYTES), dict(ws=IMG - ws_bytes()), dict(flags=8),
               dict(blur=((0, ()), (0, ())))):
        rc, err = call(**kw)
        assert rc == -2, (kw, err)


def test_aug_batch_blur_ignores_blur_arguments_without_the_flag():
    """Without YFV2_AUG_BLUR the call is yfv2_aug_batch: descriptors and workspace are not looked at."""
    torch = pytest.importorskip("torch")
    if torch.cuda.is_available():
        pytest.skip("the launch would read the fake pointers")
    rc, err = call(flags=7, blur=((7, ()), (9, ())), ws=0, nws=0)
    assert rc == -2, err


def test_workspace_size_query():
    import yfv2_engine as eng
    L = eng.lib()
    assert ws_bytes(2, 8, 8) >= IMG_BYTES + 2 * 2 * 4
    assert ws_bytes(256, 352, 352) >= 256 * 3 * 352 * 352 + 256 * 8
    nb = ctypes.c_size_t()
    for args in ((0, 8, 8), (2, 0, 8), (2, 8, 40000)):
        assert L.yfv2_aug_blur_workspace_bytes(*args, ctypes.byref(nb)) == -1
    assert L.yfv2_aug_blur_workspace_bytes(2, 8, 8, None) == -1


def test_aug_batch_still_refuses_the_blur_flag():
    import yfv2_engine as eng
    L = eng.lib()
    arr = (eng.AugParams * 2)(eng.AugParams(1.0, 0.0, 8, 8), eng.AugParams(1.0, 0.0, 8, 8))
    assert L.yfv2_aug_batch(ctypes.c_void_p(IMG), ctypes.c_void_p(OUT), 2, 8, 8, arr, ctypes.c_void_p(1), 8, None) == -1
    assert "unknown flags 0x8" in L.yfv2_last_error().decode()

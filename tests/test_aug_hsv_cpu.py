"""augment_hsv / random_resize restatement (tests/aug_hsv_oracle.py) against the real cv2 and reference goldens
(tests/golden/aug_hsv_cases.npz), the host LUT builder against the reference's LUTs, and every refusal of yfv2_aug_batch before
anything is launched."""
import ctypes
import hashlib
import os

import numpy as np
import pytest

import yfv2  # noqa: F401
import aug_hsv_cases as hc
import aug_hsv_oracle as ho


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest()


@pytest.fixture(scope="module")
def g(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "aug_hsv_cases.npz")))


def test_conversions_over_all_byte_triples_match_cv2(g):
    cube = ho.all_triples()
    hsv = ho.bgr2hsv(cube)
    assert sha(hsv) == g["bgr2hsv_sha256"].tobytes()
    assert sha(ho.hsv2bgr(cube)) == g["hsv2bgr_sha256"].tobytes()
    assert sha(ho.hsv2bgr(hsv)) == g["roundtrip_sha256"].tobytes()
    assert sha(ho.hsv2bgr(cube.reshape(-1, 1, 3))) == g["hsv2bgr_col_sha256"].tobytes()          # every pixel in cv2's tail
    assert sha(ho.hsv2bgr(cube[:, :4081].reshape(-1, 53, 3))) == g["hsv2bgr_w53_sha256"].tobytes()


def test_host_lut_builder_equals_the_reference_luts(g):
    import yfv2_engine as eng
    names = [c[0] for c in hc.HSV_CASES]
    r = np.stack([g["hsv_%s_r" % n] for n in names])
    got = eng.hsv_luts(r)
    for i, n in enumerate(names):
        assert np.array_equal(got[i], g["hsv_%s_luts" % n]), n
        assert np.array_equal(ho.hsv_luts(g["hsv_%s_r" % n]), g["hsv_%s_luts" % n]), n


@pytest.mark.parametrize("name,img_spec,u", hc.HSV_CASES, ids=[c[0] for c in hc.HSV_CASES])
def test_augment_hsv_equals_the_reference(g, name, img_spec, u):
    got = ho.augment_hsv(hc.image(*img_spec), g["hsv_%s_r" % name])
    assert sha(got) == g["hsv_%s_sha256" % name].tobytes()


def test_hsv_cases_cover_wrap_and_clip(g):
    lut = g["hsv_max_luts"]
    assert lut[0][179] < 179 and lut[0][178] < lut[0][100]            # hue wraps past 180
    assert lut[1][255] == 255 and lut[1][200] == 255 and lut[2][200] == 255   # saturation and value clip


@pytest.mark.parametrize("name,img_spec,size", hc.RESIZE_CASES, ids=[c[0] for c in hc.RESIZE_CASES])
def test_random_resize_equals_the_reference(g, name, img_spec, size):
    assert (int(g["rr_%s_rw" % name]), int(g["rr_%s_rh" % name])) == size
    assert sha(ho.random_resize(hc.image(*img_spec), *size)) == g["rr_%s_sha256" % name].tobytes()


@pytest.mark.parametrize("s", hc.RESIZE_SEEDS)
def test_random_resize_seeded_draws(g, s):
    rw, rh = int(g["rr_seed%d_rw" % s]), int(g["rr_seed%d_rh" % s])
    assert sha(ho.random_resize(hc.image(40 + s, 352, 352), rw, rh)) == g["rr_seed%d_sha256" % s].tobytes()


@pytest.mark.parametrize("s", hc.CHAIN_SEEDS)
def test_chain_equals_the_reference(g, s):
    for i, img in enumerate(hc.chain_batch(s)):
        got = ho.img_aug(img, g["chain_%d_alpha" % s][i], g["chain_%d_beta" % s][i], int(g["chain_%d_rw" % s][i]),
                         int(g["chain_%d_rh" % s][i]), g["chain_%d_r" % s][i])
        assert sha(got) == g["chain_%d_%d_sha256" % (s, i)].tobytes(), (s, i)


# ---- yfv2_aug_batch refusals: checked on the host before any launch, so this runs without a GPU ----------------------------------
def call(img=16, out=4096, N=2, H=8, W=8, params=((1.0, 0.0, 8, 8), (1.0, 0.0, 8, 8)), luts=1, flags=7):
    import yfv2_engine as eng
    L = eng.lib()
    arr = (eng.AugParams * max(len(params or ()), 1))(*[eng.AugParams(*p) for p in (params or ())])
    p = lambda v: ctypes.c_void_p(v) if v else None                        # never dereferenced: the checks come first
    rc = L.yfv2_aug_batch(p(img), p(out), N, H, W, arr if params is not None else None, p(luts), flags, None)
    return rc, L.yfv2_last_error().decode()


@pytest.mark.parametrize("kw,msg", [
    (dict(img=0), "null img"), (dict(out=0), "null img"), (dict(params=None), "params"), (dict(N=0), "N <= 0"),
    (dict(N=-3), "N <= 0"), (dict(H=0), "outside"), (dict(W=-1), "outside"), (dict(W=40000), "outside"),
    (dict(flags=8), "unknown flags"), (dict(flags=-1), "unknown flags"), (dict(luts=0), "needs luts"),
    (dict(params=((1.0, 0.0, 0, 8), (1.0, 0.0, 8, 8))), "image 0: random_resize size 0x8"),
    (dict(params=((1.0, 0.0, 8, 8), (1.0, 0.0, 8, 9))), "image 1: random_resize size 8x9"),
    (dict(params=((1.0, 0.0, 9, 8), (1.0, 0.0, 8, 8))), "image 0"),
    (dict(params=((1.0, 0.0, 8, -1), (1.0, 0.0, 8, 8))), "image 0"),
    (dict(out=16), "overlap"), (dict(out=16 + 2 * 3 * 64 - 1), "overlap"), (dict(out=16 + 1, flags=1), "overlap"),
    (dict(out=16 - 1, flags=5), "overlap"),
])
def test_aug_batch_refusals_before_any_launch(kw, msg):
    rc, err = call(**kw)
    assert rc == -1 and msg in err, (rc, err)


def test_aug_batch_refusals_accept_the_edges_without_a_device():
    """The edges that pass the checks reach the launch, which fails with YFV2_ECUDA here for want of a device."""
    torch = pytest.importorskip("torch")
    if torch.cuda.is_available():
        pytest.skip("the launch would read the fake pointers")
    for kw in (dict(params=((1.0, 0.0, 1, 1), (1.0, 0.0, 8, 8))), dict(out=16 + 2 * 3 * 64), dict(flags=0, luts=0),
               dict(flags=1, out=16)):
        rc, err = call(**kw)
        assert rc == -2, (kw, err)

"""Geometric augmentation on the host: the restatement (tests/geom_oracle.py) against the real cv2 (tests/golden/geom_cases.npz),
utils.device_aug.geometric_targets against YOLOv5's own label lines and against hand-derived boxes, the order of the draws, the
trainer's flag, and every refusal of yfv2_aug_geometric before anything is launched."""
import ctypes
import hashlib
import math
import os
import random

import numpy as np
import pytest

import yfv2  # noqa: F401
import geom_cases as gc
import geom_oracle as go


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest()


@pytest.fixture(scope="module")
def g(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "geom_cases.npz")))


def case_draws(g, name):
    return gc.unpack(g[name + "_M"], g[name + "_meta"], g[name + "_s"])


@pytest.mark.parametrize("case", gc.CASES, ids=[c[0] for c in gc.CASES])
def test_oracle_equals_cv2(g, case):
    name, N, H, W, seed = case[:5]
    got = go.augment_planar(gc.images(name, N, H, W, seed, g["jpeg_imgs"]), case_draws(g, name))
    assert sha(got) == g[name + "_sha256"].tobytes(), name
    if name + "_out" in g:
        assert np.array_equal(got, g[name + "_out"])


def test_cases_cover_the_edges(g):
    metas = {c[0]: g[c[0] + "_meta"] for c in gc.CASES}
    ends = metas["mosaic_ends"]
    assert {int(v) for v in ends[:, 5]} == {32, 96} and {int(v) for v in ends[:, 6]} == {32, 96}      # xc, yc at both ends
    assert (metas["flip_on"][:, 7] == 1).all() and (metas["flip_off"][:, 7] == 0).all()
    assert metas["ties"][:, 8].tolist() == [0, 0, 1, 1]
    assert (metas["perspective"][:, 8] == 1).all() and (metas["mosaic_n1"][:, 1:5] == 0).all()
    assert g["identity_sha256"].tobytes() == sha(gc.images("identity", 2, 48, 64, 1))          # cv2's identity warp: the input


@pytest.mark.parametrize("case", gc.CASES, ids=[c[0] for c in gc.CASES])
def test_targets_equal_yolov5s_lines(g, case):
    import utils.device_aug as da
    name, N, H, W, seed = case[:5]
    got = da.geometric_targets(gc.targets(N, seed), case_draws(g, name), H, W)
    assert got.dtype.is_floating_point and got.numpy().dtype == np.float32
    assert np.array_equal(got.numpy(), g[name + "_labels"]), name


# ---- hand-derived boxes: W = H = 100, one image, s = 1 unless stated ---------------------------------------------------------------
def one(M, box, flip=False, s=1.0, mosaic=False, src=(0, 0, 0, 0), xc=0, yc=0, perspective=False, H=100, W=100):
    import utils.device_aug as da
    d = dict(mosaic=mosaic, src=list(src), xc=xc, yc=yc, M=np.asarray(M, np.float64), perspective=perspective, flip=flip, s=s)
    t = np.array([[src[0], 7] + list(box)] if not mosaic else [[1, 7] + list(box)], np.float32)
    return da.geometric_targets(t, [d], H, W).numpy()


def shift(dx, dy=0.0):
    return [[1, 0, dx], [0, 1, dy], [0, 0, 1]]


def test_box_cut_by_the_border_is_clipped():
    r = one(shift(50), (0.4, 0.5, 0.4, 0.2))              # x 20..60 -> 70..110, clipped to 70..100 - 1e-3
    x2 = np.float32(100 - 1e-3)
    assert r.shape == (1, 6) and r[0, 1] == 7
    np.testing.assert_allclose(r[0, 2:], [(70 + x2) / 2 / 100, 0.5, (x2 - 70) / 100, 0.2], rtol=0, atol=1e-6)


def test_box_turned_45_degrees_bounds_its_corners():
    M = gc.rot(45, 1.0, 100, 100, 100, 100)
    r = one(M, (0.5, 0.5, 0.2, 0.2))
    side = 20 * math.sqrt(2) / 100
    np.testing.assert_allclose(r[0, 2:], [0.5, 0.5, side, side], rtol=0, atol=1e-5)


def test_box_dropped_by_area_thr():
    assert one(shift(-37), (0.2, 0.5, 0.4, 0.4)).shape == (0, 6)        # 40 -> 3 px wide: 0.075 of its area
    assert one(shift(-35), (0.2, 0.5, 0.4, 0.4)).shape == (1, 6)        # 5 px: 0.125


def test_box_dropped_by_wh_thr():
    assert one(np.eye(3), (0.5, 0.5, 0.02, 0.2)).shape == (0, 6)        # 2 px wide: not > 2
    assert one(np.eye(3), (0.5, 0.5, 0.025, 0.2)).shape == (1, 6)


def test_box_dropped_by_ar_thr():
    assert one(np.eye(3), (0.5, 0.5, 0.003, 0.9), H=1000, W=1000).shape == (0, 6)      # 3 x 900 px: aspect 300
    assert one(np.eye(3), (0.5, 0.5, 0.01, 0.9), H=1000, W=1000).shape == (1, 6)       # 10 x 900: aspect 90


def test_box_in_a_clipped_mosaic_tile():
    """Top-right tile with yc = H/2: rows 50..99 of image 1 land on canvas rows 0..49.  The box (local x 10..50, y 20..80) is
    clipped at the canvas top to y 0..30, and M = T @ S(0.5) @ C halves the canvas into the output."""
    M = gc.rot(0, 0.5, 200, 200, 100, 100)
    r = one(M, (0.3, 0.5, 0.4, 0.6), mosaic=True, src=(0, 1, 0, 0), xc=50, yc=50, s=0.5)
    assert r.shape == (1, 6) and r[0, 0] == 0 and r[0, 1] == 7
    np.testing.assert_allclose(r[0, 2:], [0.4, 0.075, 0.2, 0.15], rtol=0, atol=1e-6)


def test_flipped_box():
    r = one(np.eye(3), (0.3, 0.4, 0.2, 0.1), flip=True)
    np.testing.assert_allclose(r[0, 2:], [0.7, 0.4, 0.2, 0.1], rtol=0, atol=1e-6)
    assert one(np.eye(3), (0.3, 0.4, 0.2, 0.1))[0, 2] == np.float32(0.3)


def test_rows_come_out_image_by_image_in_tile_order():
    import utils.device_aug as da
    t = np.array([[0, 1, .5, .5, .2, .2], [1, 2, .5, .5, .2, .2], [1, 3, .4, .4, .2, .2], [2, 4, .5, .5, .2, .2]], np.float32)
    M = gc.rot(0, 0.5, 200, 200, 100, 100)
    d = [dict(mosaic=True, src=[2, 1, 0, 1], xc=100, yc=100, M=M, perspective=False, flip=False, s=0.5),
         dict(mosaic=False, src=[0] * 4, xc=0, yc=0, M=np.eye(3), perspective=False, flip=False, s=1.0)]
    r = da.geometric_targets(t, d, 100, 100).numpy()
    assert r[:, 0].tolist() == [0] * 6 + [1] and r[:, 1].tolist() == [4, 2, 3, 1, 2, 3, 1]


# ---- draws ------------------------------------------------------------------------------------------------------------------------
class Recorder(random.Random):
    """random.Random that logs the calls made on it (not the ones its methods make on themselves)."""
    def __init__(self, seed):
        super().__init__(seed)
        self.log, self.depth = [], 0

    def _call(self, entry, fn, *args, **kw):
        if not self.depth:
            self.log.append(entry)
        self.depth += 1
        try:
            return fn(*args, **kw)
        finally:
            self.depth -= 1

    def random(self):
        return self._call(("random",), super().random)

    def uniform(self, a, b):
        return self._call(("uniform", a, b), super().uniform, a, b)

    def choices(self, population, k=1):
        return self._call(("choices", tuple(population), k), super().choices, population, k=k)

    def shuffle(self, x):
        return self._call(("shuffle", len(x)), super().shuffle, x)


def test_draw_order():
    import utils.device_aug as da
    rng = Recorder(3)
    d = da.draw_geometric(3, 64, 96, rng, mosaic=1.0, degrees=10, translate=0.1, scale=0.5, shear=5, perspective=0.001, fliplr=0.5)
    persp = [("uniform", -0.001, 0.001)] * 2 + [("uniform", -10, 10), ("uniform", 0.5, 1.5)] + [("uniform", -5, 5)] * 2 + \
        [("uniform", 0.4, 0.6)] * 2
    one_image = [("random",), ("uniform", 32, 96), ("uniform", 48, 144), ("choices", (0, 1, 2), 3), ("shuffle", 4)] + persp + \
        [("random",)]
    log = [(e[0],) + tuple(round(v, 12) if isinstance(v, float) else v for v in e[1:]) for e in rng.log]
    assert log == one_image * 3
    assert all(i in x["src"] for i, x in enumerate(d)) and all(32 <= x["yc"] <= 96 and 48 <= x["xc"] <= 144 for x in d)
    rng = Recorder(3)
    da.draw_geometric(2, 64, 96, rng, mosaic=0.0)
    assert [e[0] for e in rng.log] == (["random"] + ["uniform"] * 8 + ["random"]) * 2


def test_draws_reproduce_random_perspective():
    """M = T @ S @ R @ P @ C as random_perspective builds it, from the same draws, with the mosaic border."""
    import utils.device_aug as da
    H, W = 64, 96
    d = da.draw_geometric(1, H, W, random.Random(9), mosaic=1.0, degrees=10, translate=0.1, scale=0.5, shear=5, perspective=0.001)[0]
    r = random.Random(9)
    r.random(); r.uniform(0, 1); r.uniform(0, 1); r.choices(range(1), k=3); r.shuffle([0, 0, 0, 0])
    C = np.eye(3); C[0, 2], C[1, 2] = -W, -H                                       # canvas 2W x 2H: its centre
    P = np.eye(3); P[2, 0] = r.uniform(-0.001, 0.001); P[2, 1] = r.uniform(-0.001, 0.001)
    a, s = r.uniform(-10, 10), r.uniform(0.5, 1.5)
    R = np.eye(3); R[:2] = [[s * math.cos(math.radians(a)), s * math.sin(math.radians(a)), 0],
                            [-s * math.sin(math.radians(a)), s * math.cos(math.radians(a)), 0]]
    S = np.eye(3); S[0, 1] = math.tan(r.uniform(-5, 5) * math.pi / 180); S[1, 0] = math.tan(r.uniform(-5, 5) * math.pi / 180)
    T = np.eye(3); T[0, 2] = r.uniform(0.4, 0.6) * W; T[1, 2] = r.uniform(0.4, 0.6) * H     # width, height = the output's
    np.testing.assert_allclose(d["M"], T @ S @ R @ P @ C, rtol=1e-12, atol=1e-12)
    assert d["s"] == s and d["perspective"]



def test_matrix_products_associate_left_to_right():
    """M is ((((T @ S) @ R) @ P) @ C), as numpy evaluates random_perspective's T @ S @ R @ P @ C, bit for bit; over 64 draws the
    other association differs in some bits, so the test sees the order."""
    import utils.device_aug as da
    H, W = 352, 352
    hyp = dict(mosaic=0.0, degrees=10, translate=0.1, scale=0.5, shear=5, perspective=0.001, fliplr=0.5)
    draws = da.draw_geometric(64, H, W, random.Random(4), **hyp)

    def mm(x, y):                                      # one product, each entry summed in index order in Python floats
        return [[x[i][0] * y[0][j] + x[i][1] * y[1][j] + x[i][2] * y[2][j] for j in range(3)] for i in range(3)]
    r, differs = random.Random(4), 0
    for d in draws:
        r.random()
        C = [[1, 0, -W / 2], [0, 1, -H / 2], [0, 0, 1]]
        P = [[1, 0, 0], [0, 1, 0], [r.uniform(-0.001, 0.001), r.uniform(-0.001, 0.001), 1]]
        a, s = r.uniform(-10, 10), r.uniform(0.5, 1.5)
        al, be = math.cos(a * (math.pi / 180)) * s, math.sin(a * (math.pi / 180)) * s
        R = [[al, be, 0], [-be, al, 0], [0, 0, 1]]
        S = [[1, math.tan(r.uniform(-5, 5) * math.pi / 180), 0], [math.tan(r.uniform(-5, 5) * math.pi / 180), 1, 0], [0, 0, 1]]
        T = [[1, 0, r.uniform(0.4, 0.6) * W], [0, 1, r.uniform(0.4, 0.6) * H], [0, 0, 1]]
        r.random()
        assert np.array_equal(d["M"], np.array(mm(mm(mm(mm(T, S), R), P), C)))
        differs += not np.array_equal(d["M"], np.array(mm(T, mm(S, mm(R, mm(P, C))))))
    assert differs > 0


def test_targets_over_the_batch_equal_image_by_image():
    """geometric_targets gathers every tile's rows once and runs each step over the whole batch: the same rows and bits as
    calling it for each output image alone."""
    import utils.device_aug as da
    for seed in range(40):
        rs = np.random.RandomState(seed)
        N, (H, W) = int(rs.randint(1, 10)), [(64, 64), (352, 352), (192, 320)][seed % 3]
        d = da.draw_geometric(N, H, W, random.Random(seed), mosaic=0.5, degrees=30, translate=0.2, scale=0.5, shear=5,
                              perspective=0.001 * (seed % 2), fliplr=0.5)
        t = np.array([[n, rs.randint(0, 80), rs.uniform(-0.1, 1.1), rs.uniform(-0.1, 1.1), rs.uniform(0.001, 0.8),
                       rs.uniform(0.001, 0.8)] for n in range(N) for _ in range(rs.randint(0, 6))], np.float32).reshape(-1, 6)
        whole = da.geometric_targets(t, d, H, W).numpy()
        each = []
        for n in range(N):
            r = da.geometric_targets(t, [d[n]], H, W).numpy()
            r[:, 0] = n
            each.append(r)
        assert np.array_equal(whole, np.concatenate(each)), seed


def test_geometric_batch_rejects_unknown_hyperparameters():
    import utils.device_aug as da
    with pytest.raises(TypeError, match="flipud"):
        da.geometric_batch(None, None, flipud=0.5)


def test_trainer_flag_needs_device_aug_and_known_keys():
    import train_dist
    for argv in (["--device-aug-geom"], ["--device-aug", "--device-aug-geom", "flipud=0.5"],
                 ["--device-aug", "--device-aug-geom", "mosaic=x"], ["--device-aug", "--device-aug-geom", "mosaic"]):
        with pytest.raises(SystemExit) as e:
            train_dist.main(argv)
        assert e.value.code == 2, argv


# ---- yfv2_aug_geometric refusals: checked on the host before any launch, so this runs without a GPU -------------------------------
BASE = 1 << 20
SHIFT = ((1, 0, 3), (0, 1, -2), (0, 0, 1))


def geom(M=SHIFT, perspective=0, mosaic=0, src=(0, 0, 0, 0), xc=8, yc=8, flip=0):
    import yfv2_engine as eng
    d = eng.AugGeom()
    d.m[:] = [float(v) for row in M for v in row]
    d.perspective, d.mosaic, d.flip, d.xc, d.yc = perspective, mosaic, flip, xc, yc
    d.src[:] = list(src)
    return d


def call(img=BASE, out=BASE * 4, N=2, H=8, W=8, params="default"):
    import yfv2_engine as eng
    L = eng.lib()
    if params == "default":
        params = [geom(), geom(src=(1, 0, 0, 0))]
    arr = (eng.AugGeom * max(len(params or ()), 1))(*(params or ()))
    p = lambda v: ctypes.c_void_p(v) if v else None                        # never dereferenced: the checks come first
    rc = L.yfv2_aug_geometric(p(img), p(out), N, H, W, arr if params is not None else None, None)
    return rc, L.yfv2_last_error().decode()


def bad(**kw):
    return [geom(), geom(**kw)]


@pytest.mark.parametrize("kw,msg", [
    (dict(img=0), "null img"), (dict(out=0), "null img"), (dict(params=None), "params"), (dict(N=0), "N <= 0"),
    (dict(N=-1), "N <= 0"), (dict(H=0), "outside 1..32768"), (dict(W=-2), "outside 1..32768"), (dict(W=32769), "outside 1..32768"),
    (dict(out=BASE), "overlap"), (dict(out=BASE + 2 * 3 * 64 - 1), "overlap"), (dict(out=BASE - 2 * 3 * 64 + 1), "overlap"),
    (dict(params=bad(perspective=2)), "image 1: perspective, mosaic and flip must be 0 or 1"),
    (dict(params=bad(mosaic=-1)), "must be 0 or 1"), (dict(params=bad(flip=2)), "must be 0 or 1"),
    (dict(params=bad(src=(2, 0, 0, 0))), "image 1: src[0] = 2 outside [0, 2)"),
    (dict(params=bad(src=(-1, 0, 0, 0))), "src[0] = -1"),
    (dict(params=bad(mosaic=1, src=(0, 1, 0, 2))), "src[3] = 2"),
    (dict(params=bad(mosaic=1), H=7, W=8), "mosaic needs even H and W"), (dict(params=bad(mosaic=1), W=9), "even H and W"),
    (dict(params=bad(mosaic=1, xc=3)), "mosaic centre (3, 8) outside [4, 12] x [4, 12]"),
    (dict(params=bad(mosaic=1, xc=13)), "mosaic centre"), (dict(params=bad(mosaic=1, yc=3)), "mosaic centre"),
    (dict(params=bad(mosaic=1, yc=13)), "mosaic centre"),
    (dict(params=bad(M=((1, 2, 0), (2, 4, 0), (0, 0, 1)))), "image 1: singular matrix"),
    (dict(params=bad(M=((1, 2, 0), (2, 4, 0), (0, 0, 1)), perspective=1)), "singular matrix"),
    (dict(params=bad(M=((1, 0, float("nan")), (0, 1, 0), (0, 0, 1)))), "matrix entries must be finite"),
    (dict(params=bad(M=((1, 0, 0), (0, 1, 0), (0, 0, float("inf"))), perspective=1)), "finite"),
    (dict(params=bad(M=((1e-7, 0, 0), (0, 1, 0), (0, 0, 1)))), "2^30"),
    (dict(params=bad(M=((1e-155, 0, 0), (0, 1e-155, 0), (0, 0, 1)), perspective=1)), "the inverse has non-finite entries"),
    (dict(H=32767), "image 0: image canvas 8x32767: its sides must be below 32767"),
    (dict(W=32768), "canvas 32768x8"), (dict(params=bad(mosaic=1), W=16384), "image 1: mosaic canvas 32768x16"),
    (dict(params=bad(mosaic=1), H=16384), "mosaic canvas 16x32768"),
])
def test_aug_geometric_refusals_before_any_launch(kw, msg):
    rc, err = call(**kw)
    assert rc == -1 and msg in err, (rc, err)


def test_aug_geometric_refusals_accept_the_edges_without_a_device():
    """The edges that pass the checks reach the launch, which fails with YFV2_ECUDA here for want of a device."""
    torch = pytest.importorskip("torch")
    if torch.cuda.is_available():
        pytest.skip("the launch would read the fake pointers")
    for kw in (dict(out=BASE + 2 * 3 * 64), dict(out=BASE - 2 * 3 * 64), dict(params=bad(mosaic=1, xc=4, yc=12)),
               dict(params=bad(mosaic=1, xc=12, yc=4, src=(1, 1, 0, 1))), dict(params=bad(src=(1, 5, -3, 9))),
               dict(params=bad(flip=1, perspective=1, M=((1, 0, 0), (0, 1, 0), (0.001, 0, 1)))), dict(H=1, W=1),
               dict(H=32766), dict(W=16382, params=bad(mosaic=1, xc=8191)), dict(H=16382, params=bad(mosaic=1, yc=8191))):
        rc, err = call(**kw)
        assert rc == -2, (kw, err)


def test_descriptor_layout():
    import yfv2_engine as eng
    assert ctypes.sizeof(eng.AugGeom) == 112
    assert [getattr(eng.AugGeom, f).offset for f in ("m", "perspective", "mosaic", "src", "xc", "yc", "flip")] == \
        [0, 72, 76, 80, 96, 100, 104]

"""The JPEG encode without a GPU: tests/jpeg_enc_harness.cu (yfv2_jpeg_encode_plan's headers, then jpeg_enc.cuh's per-block
functions composed one block at a time) against cv2.imencode's bytes frozen in tests/golden/jpeg_encode_cases.npz, a live sweep
against cv2 where it is importable, and the plan's refusals."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

import yfv2  # noqa: F401
import jpeg_encode_cases as C
import yfv2_engine as eng

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "jpeg_encode_cases.npz")
NVCC = "/usr/local/cuda/bin/nvcc"


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
    if nvcc is None:
        pytest.skip("no nvcc")
    d = tmp_path_factory.mktemp("jpeg_enc_harness")
    exe = str(d / "harness")
    subprocess.run([nvcc, "-std=c++17", "-O1", "-Wno-deprecated-gpu-targets", "-diag-suppress", "20011", "-gencode",
                    "arch=compute_90a,code=sm_90a", os.path.join(ROOT, "tests", "jpeg_enc_harness.cu"), "-o", exe],
                   check=True, capture_output=True)
    return exe, d


def encode(harness, img, params):
    exe, d = harness
    img = np.ascontiguousarray(img)
    img.tofile(str(d / "in.raw"))
    ch = 1 if img.ndim == 2 else 3
    r = subprocess.run([exe, str(d / "in.raw"), str(img.shape[1]), str(img.shape[0]), str(ch), str(d / "out.jpg")]
                       + [str(p) for p in params], capture_output=True, text=True, check=True)
    status = int(r.stdout.split()[0])
    return status, (open(d / "out.jpg", "rb").read() if status == 0 else r.stdout)


def case_params(c):
    return [1, c["quality"], 7, eng.JPEG_SAMPLING[c["sampling"]], 4, c["restart"]]


def sos_end(b):
    """Length of the headers: everything up to the end of the SOS segment"""
    i = 2
    while True:
        n = b[i + 2] << 8 | b[i + 3]
        if b[i + 1] == 0xDA:
            return i + 2 + n
        i += 2 + n


def test_cases_without_cv2_match_the_golden(harness):
    """bgr and grey cases need no conversion: the harness's files equal cv2's, headers first"""
    g = np.load(GOLDEN)
    n = 0
    for c in C.cases():
        if c["photo"] or c["layout"] not in ("bgr", "gray") or c["name"] not in g:
            continue
        img = C.frame(c["layout"], c["w"], c["h"], c["kind"], c["seed"])
        if c["region"]:
            x0, y0, w, h = c["region"]
            img = img[y0:y0 + h, x0:x0 + w]
        want = g[c["name"]].tobytes()
        st, got = encode(harness, img, case_params(c))
        assert st == 0, got
        assert got[:sos_end(want)] == want[:sos_end(want)], c["name"] + ": headers"
        assert got == want, c["name"]
        n += 1
    assert n > 150


def test_converted_cases_match_the_golden(harness):
    cv2 = pytest.importorskip("cv2")
    import importlib.util
    spec = importlib.util.spec_from_file_location("mk", os.path.join(ROOT, "tests", "golden", "make_golden_jpeg_encode.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    g = np.load(GOLDEN)
    for c in C.cases():
        if c["name"] not in g or (c["layout"] in ("bgr", "gray") and not c["photo"]):
            continue
        st, got = encode(harness, mk.image(c), case_params(c))
        assert st == 0 and got == g[c["name"]].tobytes(), c["name"]
    del cv2


def test_live_sweep_against_cv2(harness):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.RandomState(2024)
    bad = []
    for it in range(3000):
        w, h = int(rng.randint(1, 90)), int(rng.randint(1, 90))
        kind = ["noise", "flat0", "flat255", "edges", "checker"][rng.randint(5)]
        img = C.content(kind, w, h, it)
        if rng.rand() < 0.25:
            img = np.ascontiguousarray(img[:, :, 0])
        params = [cv2.IMWRITE_JPEG_QUALITY, int(rng.randint(-10, 111)), cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                  int(rng.choice([0x221111, 0x211111, 0x111111])), cv2.IMWRITE_JPEG_RST_INTERVAL,
                  int(rng.choice([0, 0, 1, 2, 3, 5, 17, 70000, -3]))]
        st, got = encode(harness, img, params)
        if st != 0 or got != cv2.imencode(".jpg", img, params)[1].tobytes():
            bad.append((w, h, kind, img.ndim, params))
    assert not bad, bad[:5]


def _plan(srcs):
    L = eng.lib()
    arr = (eng.JpegEncSrc * len(srcs))(*srcs)
    mb, wb, ab = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_size_t()
    rc = L.yfv2_jpeg_encode_plan(arr, len(srcs), None, 0, ctypes.byref(mb), ctypes.byref(wb), None, ctypes.byref(ab))
    return rc, L.yfv2_last_error().decode()


def _src(w=64, h=48, params=(), region=None, kind=0):
    s = eng.JpegEncSrc()
    s.kind = kind
    s.f.bgr.data, s.f.bgr.w, s.f.bgr.h, s.f.bgr.pitch = 4096, w, h, 3 * w   # the plan never reads the pixels
    s.x0, s.y0, s.w, s.h = region or (0, 0, w, h)
    s._p = (ctypes.c_int * max(1, len(params)))(*params)
    s.params, s.nparams = ctypes.cast(s._p, ctypes.POINTER(ctypes.c_int)), len(params)
    return s


@pytest.mark.parametrize("params,code,what", [
    ((3, 1), -3, "IMWRITE_JPEG_OPTIMIZE"), ((2, 1), -3, "IMWRITE_JPEG_PROGRESSIVE"), ((5, 40), -3, "IMWRITE_JPEG_LUMA_QUALITY"),
    ((6, 40), -3, "IMWRITE_JPEG_CHROMA_QUALITY"), ((7, 0x121111), -3, "4:4:0"), ((7, 0x411111), -3, "4:1:1"),
    ((7, 0x123456), -1, "sampling factor"), ((1,), -1, "pairs")])
def test_refused_params(params, code, what):
    rc, err = _plan([_src(), _src(params=params)])
    assert rc == code and "output 1" in err and what in err, err


def test_params_cv2_leaves_alone_are_accepted():
    assert _plan([_src(params=(3, 0, 2, 0, 5, -1, 6, -1, 16, 9))])[0] == 0


@pytest.mark.parametrize("region", [(0, 0, 0, 5), (0, 0, 5, 0), (60, 0, 5, 5), (0, 45, 5, 5), (-1, 0, 5, 5), (64, 48, 1, 1)])
def test_refused_regions(region):
    rc, err = _plan([_src(region=region)])
    assert rc == -1 and "output 0" in err and "region" in err, err


def test_refused_sizes():
    rc, err = _plan([_src(w=40000, h=8)])
    assert rc == -3 and "output 0" in err and "32768" in err, err
    assert _plan([_src(w=32768, h=2)])[0] == 0


def test_refused_frames():
    s = _src()
    s.f.bgr.data = None
    rc, err = _plan([s])
    assert rc == -1 and "output 0" in err and "null" in err, err

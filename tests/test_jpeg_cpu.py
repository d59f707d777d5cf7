"""JPEG decode without a GPU: the host parser (yfv2_jpeg_parse through ctypes) on every fixture of tests/jpeg_cases.py, and a CPU
build of the decode's own functions (csrc/jpeg.cuh, compiled with nvcc into tests/jpeg_harness.cu) against cv2's bytes."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import yfv2  # noqa: F401  (registers the package dir)
import jpeg_cases as jc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "jpeg_cases.npz"))


def test_parser_accepts_every_supported_fixture(golden):
    import yfv2_engine
    files = [golden["jpg_" + c[0]] for c in jc.CASES]
    infos, blob, (ws, fr), _, _ = yfv2_engine.parse_jpeg(files, [c[0] for c in jc.CASES], blob=True)
    offset = 0
    for case, info in zip(jc.CASES, infos):
        name, _, (h, w), s, _, _, rst, orient, _ = case
        assert info["status"] == 0 and info["reason"] == "", name
        assert (info["h"], info["w"], 3) == jc.golden_shape(golden, name), name
        swap = orient is not None and orient >= 5
        assert (info["h"], info["w"]) == ((w, h) if swap else (h, w)), name
        assert info["components"] == (1 if s == "grey" else 3), name
        assert (info["h_samp"], info["v_samp"]) == jc.SAMPLINGS[s], name
        assert info["restart_interval"] == rst and info["segments"] == jc.segments(case), name
        assert info["orientation"] == (orient or 1), name
        assert info["frame_offset"] == offset, name
        offset = (offset + 3 * h * w + 15) // 16 * 16
    assert fr == offset and ws > 0 and blob.numel() > 0


@pytest.mark.parametrize("name,code,reason", jc.UNSUPPORTED, ids=[u[0] for u in jc.UNSUPPORTED])
def test_parser_refuses_unsupported_files_with_their_reason(golden, name, code, reason):
    import yfv2_engine
    good = golden["jpg_q75_420_opt0"]
    with pytest.raises(yfv2_engine.Yfv2Error, match=r"1 of 2 files refused: bad\.jpg: .*%s" % reason):
        yfv2_engine.parse_jpeg([good, golden["bad_" + name]], ["good.jpg", "bad.jpg"])
    import ctypes
    L = yfv2_engine.lib()
    buf = golden["bad_" + name]
    info = yfv2_engine.JpegInfo()
    off = (ctypes.c_longlong * 2)(0, buf.size)
    sz = ctypes.c_size_t()
    assert L.yfv2_jpeg_parse(buf.ctypes.data, off, 1, ctypes.byref(info), None, 0, ctypes.byref(sz), ctypes.byref(sz), ctypes.byref(sz)) == code
    assert info.status == code and reason in info.reason.decode() and reason in L.yfv2_last_error().decode()


def test_parse_and_decode_refuse_bad_arguments(golden):
    import ctypes
    import yfv2_engine
    L = yfv2_engine.lib()
    buf = golden["jpg_q75_420_opt0"]
    info = yfv2_engine.JpegInfo()
    sz = [ctypes.c_size_t() for _ in range(3)]
    ref = [ctypes.byref(s) for s in sz]
    off = (ctypes.c_longlong * 2)(0, buf.size)
    assert L.yfv2_jpeg_parse(None, off, 1, ctypes.byref(info), None, 0, *ref) == -1
    assert L.yfv2_jpeg_parse(buf.ctypes.data, (ctypes.c_longlong * 2)(5, 2), 1, ctypes.byref(info), None, 0, *ref) == -1
    assert b"ascending" in L.yfv2_last_error()
    assert L.yfv2_jpeg_parse(buf.ctypes.data, off, 1, ctypes.byref(info), None, 0, *ref) == 0
    blob = (ctypes.c_uint8 * sz[0].value)()
    assert L.yfv2_jpeg_parse(buf.ctypes.data, off, 1, ctypes.byref(info), blob, sz[0].value - 1, *ref) == -4
    assert L.yfv2_jpeg_parse(buf.ctypes.data, off, 1, ctypes.byref(info), blob, sz[0].value, *ref) == 0
    meta, ws, fr = (s.value for s in sz)
    fake = ctypes.c_void_p(16)                                           # never dereferenced: every check comes first
    args = lambda m=meta, fb=buf.size, frb=fr, wsb=ws, ph=7, mh=blob: (mh, fake, m, fake, fb, fake, frb, fake, fake, wsb, ph, None)  # noqa: E731
    for kw, what in [({"m": meta - 1}, b"blob"), ({"fb": buf.size - 1}, b"files_bytes"), ({"frb": fr - 1}, b"frames_bytes"),
                     ({"wsb": ws - 1}, b"workspace_bytes"), ({"ph": 0}, b"phases"), ({"ph": 8}, b"phases")]:
        assert L.yfv2_jpeg_decode(*args(**kw)) == -1, kw
        assert what in L.yfv2_last_error(), (kw, L.yfv2_last_error())
    junk = (ctypes.c_uint8 * meta)()
    assert L.yfv2_jpeg_decode(*args(mh=junk)) == -1 and b"not a blob" in L.yfv2_last_error()


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    """tests/jpeg_harness.cu built for the host with the parser compiled in (address-sanitised where the toolchain supports it;
    otherwise a plain build, which still compares bytes but no longer sees reads past a file's end)."""
    if not os.path.exists(NVCC) and shutil.which("nvcc") is None:
        pytest.skip("no nvcc")
    nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
    d = tmp_path_factory.mktemp("jpeg_harness")
    exe = str(d / "harness")
    base = [nvcc, "-std=c++17", "-O1", "-Wno-deprecated-gpu-targets", "-gencode", "arch=compute_90a,code=sm_90a",
            os.path.join(ROOT, "tests", "jpeg_harness.cu"), "-o", exe]
    r = subprocess.run(base[:4] + ["-Xcompiler", "-fsanitize=address", "-Xlinker", "-lasan"] + base[4:], capture_output=True, text=True)
    if r.returncode != 0:
        subprocess.run(base, check=True, capture_output=True)
    return exe, d


def run_harness(harness, items):
    exe, d = harness
    args = []
    for name, buf in items:
        src, dst = str(d / (name + ".jpg")), str(d / (name + ".bgr"))
        buf.tofile(src)
        args += [src, dst]
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0")
    r = subprocess.run([exe] + args, capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr[-3000:]
    lines = r.stdout.strip().splitlines()
    assert len(lines) == len(items)
    return [tuple(int(v) for v in ln.split()[:4]) for ln in lines], [str(d / (n + ".bgr")) for n, _ in items]


def test_cpu_build_of_the_decode_equals_cv2_on_every_fixture(golden, harness):
    items = [(c[0], golden["jpg_" + c[0]]) for c in jc.CASES]
    results, outs = run_harness(harness, items)
    bad = []
    for (name, _), (status, w, h, err), out in zip(items, results, outs):
        assert (status, err) == (0, 0), name
        got = np.fromfile(out, np.uint8)
        if got.size != 3 * h * w or not jc.equals_golden(golden, name, got.reshape(h, w, 3)):
            bad.append(name)
    assert not bad, "differ from cv2: %s" % bad


def test_cpu_build_on_the_reference_photos(golden_dir, harness):
    frames = np.load(os.path.join(golden_dir, "frames_modelzoo.npz"))
    items = [(s, np.fromfile(os.path.join(golden_dir, s + ".jpg"), np.uint8)) for s in ("000139", "000004")]
    results, outs = run_harness(harness, items)
    for (s, _), (status, w, h, err), out in zip(items, results, outs):
        assert (status, err, (h, w)) == (0, 0, frames[s].shape[:2])
        assert np.array_equal(np.fromfile(out, np.uint8).reshape(frames[s].shape), frames[s]), s


def test_truncated_scan_is_flagged_without_reading_past_the_file(golden, harness):
    """A file cut inside its entropy-coded data parses (libjpeg decodes what is there) and the decode pads with zero bits and flags
    it; the harness holds the file in a buffer of exactly its size, under AddressSanitizer when available."""
    buf = golden["cut_" + jc.TRUNCATED_SCAN]
    (status, w, h, err), = run_harness(harness, [("cut", buf)])[0]
    assert status == 0 and (w, h) == (96, 64) and err & 1

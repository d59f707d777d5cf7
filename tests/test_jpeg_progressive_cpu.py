"""Progressive JPEG files (tests/jpeg_progressive_cases.py) through the host parser (yfv2_jpeg_parse_ex) and the address-sanitised
CPU build of the decode (tests/jpeg_progressive_harness.cu), against what cv2.imdecode made of each.  The contract: with
YFV2_JPEG_PROGRESSIVE a file the decoder accepts and does not flag is cv2's frame byte for byte; only damaged scans are flagged,
and every file cv2 returns no image for is refused or flagged; a refused file names why; nothing is read past a file's end.
Without the flag every progressive file is refused as before."""
import ctypes
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

import yfv2  # noqa: F401  (registers the package dir)
import jpeg_cases as jc
import jpeg_progressive_cases as pc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ACCEPTED = [n for n in pc.CASES if n not in pc.REFUSED]


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "jpeg_progressive.npz"))


def parse_one(buf, flags=1):
    import yfv2_engine
    L = yfv2_engine.lib()
    info = yfv2_engine.JpegInfo()
    sz = [ctypes.c_size_t() for _ in range(3)]
    off = (ctypes.c_longlong * 2)(0, buf.size)
    rc = L.yfv2_jpeg_parse_ex(buf.ctypes.data, off, 1, flags, ctypes.byref(info), None, 0, *[ctypes.byref(s) for s in sz])
    return rc, info


def script(buf):
    """(frame (w, h, [(id, h, v)]), [(component ids, ss, se, ah, al, restart interval)]) read from a file's markers: a restatement
    of the parse, for the scan, segment and level counts."""
    b, pos, scans, rst, frame = bytes(buf), 2, [], 0, None
    while pos + 4 <= len(b):
        m = b[pos + 1]
        if m == 0xD9:
            break
        n = struct.unpack(">H", b[pos + 2:pos + 4])[0]
        p = b[pos + 4:pos + 2 + n]
        pos += 2 + n
        if m == 0xC2:
            frame = (struct.unpack(">H", p[3:5])[0], struct.unpack(">H", p[1:3])[0], [(p[6 + 3 * c], p[7 + 3 * c] >> 4, p[7 + 3 * c] & 15)
                                                                                      for c in range(p[5])])
        elif m == 0xDD:
            rst = struct.unpack(">H", p[:2])[0]
        elif m == 0xDA:
            ns = p[0]
            scans.append(([p[1 + 2 * k] for k in range(ns)], p[1 + 2 * ns], p[2 + 2 * ns], p[3 + 2 * ns] >> 4, p[3 + 2 * ns] & 15, rst))
            while True:
                pos = b.index(b"\xff", pos)
                if b[pos + 1] == 0 or 0xD0 <= b[pos + 1] <= 0xD7:
                    pos += 2
                    continue
                break
    return frame, scans


def expected_counts(buf):
    """(scans, segments, levels) of an undamaged progressive file"""
    (w, h, comps), scans = script(buf)
    grey = len(comps) == 1
    hmax = 1 if grey else max(c[1] for c in comps)
    vmax = 1 if grey else max(c[2] for c in comps)
    mcus = -(-w // (8 * hmax)) * -(-h // (8 * vmax))
    levels, segs = [], 0
    for i, (ids, ss, se, ah, al, rst) in enumerate(scans):
        if len(ids) > 1:
            units = mcus
        else:
            _, ch, cv = next(c for c in comps if c[0] == ids[0])
            ch, cv = (1, 1) if grey else (ch, cv)
            units = -(-(-(-w * ch // hmax)) // 8) * -(-(-(-h * cv // vmax)) // 8)
        segs += -(-units // rst) if rst else 1
        lv = 0
        for j in range(i):
            if set(ids) & set(scans[j][0]) and scans[j][1] <= se and ss <= scans[j][2]:
                lv = max(lv, levels[j] + 1)
        levels.append(lv)
    return len(scans), segs, max(levels) + 1


def test_goldens_hold_every_case(golden):
    assert sorted(k[4:] for k in golden.files if k.startswith("jpg_")) == sorted(pc.CASES)
    for name in pc.CASES:
        assert ("none_" + name in golden.files) != ("shape_" + name in golden.files), name
    assert set(pc.DAMAGED) <= set(pc.CASES) and set(pc.REFUSED) <= set(pc.CASES)


def test_parser_accepts_or_refuses_each_case_with_its_reason(golden):
    wrong = []
    for name in pc.CASES:
        rc, info = parse_one(golden["jpg_" + name])
        if name in pc.REFUSED:
            code, reason = pc.REFUSED[name]
            if (rc, info.status) != (code, code) or reason not in info.reason.decode():
                wrong.append((name, rc, info.reason.decode()))
        elif rc != 0:
            wrong.append((name, rc, info.reason.decode()))
        elif "shape_" + name in golden.files and (info.h, info.w, 3) != jc.golden_shape(golden, name):
            wrong.append((name, "size", info.h, info.w))
    assert not wrong, wrong


def test_scan_segment_and_level_counts(golden, harness):
    names = [n for n in ACCEPTED if n not in pc.DAMAGED]
    results, _ = run_harness(harness, [(n, golden["jpg_" + n]) for n in names])
    wrong = []
    for name, (status, w, h, err, scans, levels) in zip(names, results):
        _, info = parse_one(golden["jpg_" + name])
        want = expected_counts(golden["jpg_" + name])
        if (info.scans, info.segments, levels) != want or scans != info.scans:
            wrong.append((name, (info.scans, info.segments, levels), want))
    assert not wrong, wrong
    # libjpeg's default script: 10 scans over 3 levels (DC and first AC bands; Y's second band and the refinements of DC and
    # chroma; Y's last refinement), 6 scans for grey
    cv2 = dict(zip(names, results))
    assert cv2["cv2_q50_420"][4:] == (10, 3) and cv2["cv2_q50_grey"][4] == 6
    assert cv2["script_grey_wide"][4] == 77                            # a DC chain from Al 13 and 63 1-wide bands


def test_baseline_files_keep_one_scan_under_the_flag(golden_dir):
    base = np.load(os.path.join(golden_dir, "jpeg_cases.npz"))
    for c in jc.CASES[:20]:
        rc, info = parse_one(base["jpg_" + c[0]])
        assert (rc, info.scans, info.segments) == (0, 1, jc.segments(c)), c[0]


def test_without_the_flag_progressive_files_are_refused_as_before(golden):
    for name in pc.CASES:
        buf = golden["jpg_" + name]
        if name == "bad_sof10":
            continue
        rc, info = parse_one(buf, flags=0)
        assert (rc, info.status) == (-3, -3) and info.reason.decode() == "progressive DCT (SOF2)", name
    import yfv2_engine
    with pytest.raises(yfv2_engine.Yfv2Error, match=r"b\.jpg: progressive DCT \(SOF2\)"):
        yfv2_engine.parse_jpeg([golden["jpg_enc_base"]], ["b.jpg"])
    infos, *_ = yfv2_engine.parse_jpeg([golden["jpg_enc_base"]], progressive=True)
    assert infos[0]["scans"] == 10 and infos[0]["status"] == 0


def test_existing_sof2_fixture_stays_refused_under_the_flag(golden_dir):
    base = np.load(os.path.join(golden_dir, "jpeg_cases.npz"))
    rc, info = parse_one(base["bad_sof2"])
    assert rc == -1 and "a DC scan with Se = 63" in info.reason.decode()
    rc, info = parse_one(base["bad_progressive"])
    assert rc == 0 and info.scans == 10


def test_bad_flags_are_refused(golden):
    import yfv2_engine
    buf = golden["jpg_enc_base"]
    for flags in (2, 3, -1, 1 << 30):
        rc, _ = parse_one(buf, flags)
        assert rc == -1 and b"flags" in yfv2_engine.lib().yfv2_last_error(), flags


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    """tests/jpeg_progressive_harness.cu built for the host with the parser compiled in (address-sanitised where the toolchain
    supports it, as tests/test_jpeg_cpu.py builds tests/jpeg_harness.cu)."""
    if not os.path.exists(NVCC) and shutil.which("nvcc") is None:
        pytest.skip("no nvcc")
    nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
    d = tmp_path_factory.mktemp("jpeg_progressive_harness")
    exe = str(d / "harness")
    base = [nvcc, "-std=c++17", "-O1", "-Wno-deprecated-gpu-targets", "-gencode", "arch=compute_90a,code=sm_90a",
            os.path.join(ROOT, "tests", "jpeg_progressive_harness.cu"), "-o", exe]
    r = subprocess.run(base[:4] + ["-Xcompiler", "-fsanitize=address", "-Xlinker", "-lasan"] + base[4:], capture_output=True, text=True)
    if r.returncode != 0:
        subprocess.run(base, check=True, capture_output=True)
    return exe, d


def run_harness(harness, items):
    """[(status, w, h, flags, scans, levels)] and the output paths of the harness run on items [(name, bytes)]"""
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
    return [tuple(int(v) for v in ln.split()[:6]) for ln in lines], [str(d / (n + ".bgr")) for n, _ in items]


def test_cpu_build_equals_cv2_unless_damaged(golden, harness):
    items = [(n, golden["jpg_" + n]) for n in pc.CASES]
    results, outs = run_harness(harness, items)                       # a read past a file's end fails the harness run
    differ, unflagged_none, flagged_clean, refused = [], [], [], []
    for (name, _), (status, w, h, err, _, _), out in zip(items, results, outs):
        if status != 0:
            if name not in pc.REFUSED:
                refused.append(name)
            continue
        if err and name not in pc.DAMAGED:
            flagged_clean.append((name, err))
        if "none_" + name in golden.files:
            if not err:
                unflagged_none.append(name)
            continue
        got = np.fromfile(out, np.uint8)
        if not err and (got.size != 3 * h * w or not jc.equals_golden(golden, name, got.reshape(h, w, 3))):
            differ.append(name)
    assert not refused, "refused: %s" % refused
    assert not differ, "unflagged and different from cv2: %s" % differ
    assert not unflagged_none, "cv2 cannot decode these, the decode does not flag them: %s" % unflagged_none
    assert not flagged_clean, "flagged though undamaged: %s" % flagged_clean


def test_damaged_files_are_flagged_with_their_cause(golden, harness):
    items = [(n, golden["jpg_" + n]) for n in pc.DAMAGED]
    results, _ = run_harness(harness, items)
    flags = {n: r[3] for (n, _), r in zip(items, results)}
    for n in pc.DAMAGED:
        if n.startswith("cut_"):
            assert flags[n] & 1, n                                     # cv2.imdecode returns no image for a file cut before EOI
    assert flags["rst_renumbered_in_refinement"] & 4
    assert flags["corrupt_run_past_band"] & 2                          # a run past its band writes outside it


def test_lossless_recodes_of_the_photos_equal_their_golden_frames(golden, golden_dir, harness):
    """The photos re-coded as progressive files with their own coefficients decode to cv2.imread's frames of the originals, by
    cv2's script and by a seeded script with AC approximation chains."""
    frames = np.load(os.path.join(golden_dir, "frames_modelzoo.npz"))
    items = [("tx_%s_%s" % (k, s), golden["jpg_tx_%s_%s" % (k, s)]) for s in pc.PHOTOS for k in ("cv2", "seeded")]
    results, outs = run_harness(harness, items)
    for (name, _), (status, w, h, err, scans, _), out in zip(items, results, outs):
        s = name[-6:]
        assert (status, err, (h, w)) == (0, 0, frames[s].shape[:2]), name
        assert scans == 10 if "_cv2_" in name else scans > 10, name
        assert np.array_equal(np.fromfile(out, np.uint8).reshape(frames[s].shape), frames[s]), name

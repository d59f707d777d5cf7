"""The files of tests/jpeg_foreign_cases.py decoded on the device (JpegBatch: yfv2_jpeg_parse + yfv2_jpeg_decode), one file per call
and once as a shuffled batch mixed with the jpeg_cases fixtures.  On every file the parser accepts, damaged and flagged ones
included, the device's bytes and flags equal the CPU build of the same functions (tests/jpeg_harness.cu); on unflagged files the
bytes are cv2's.  test_jpeg_foreign_cpu.py runs the same files under AddressSanitizer first."""
import os

import numpy as np
import pytest

import yfv2  # noqa: F401
import jpeg_cases as jc
import jpeg_foreign_cases as fc
import yfv2_engine as eng
from test_jpeg_cpu import harness, run_harness  # noqa: F401  (the harness fixture)

pytestmark = pytest.mark.gpu

ACCEPTED = [n for n in fc.CASES if n not in fc.REFUSED]


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "jpeg_foreign.npz"))


@pytest.fixture(scope="module")
def host(golden, harness):  # noqa: F811
    """name -> (flags, BGR bytes) of the CPU build"""
    items = [(n, golden["jpg_" + n]) for n in ACCEPTED]
    results, outs = run_harness(harness, items)
    out = {}
    for (name, _), (status, w, h, err), path in zip(items, results, outs):
        assert status == 0, name
        out[name] = (err, np.fromfile(path, np.uint8).reshape(h, w, 3))
    return out


def device_decode(files):
    b = eng.JpegBatch(files, "cuda")
    b.decode()
    return [f.cpu().numpy() for f in b.frames()], b.errors.cpu().tolist()


def check(golden, host, name, got, err, bad):
    herr, hbytes = host[name]
    if err != herr or not np.array_equal(got, hbytes):
        bad.append((name, "device != host build", err, herr))
    elif not err and "none_" + name in golden.files:
        bad.append((name, "cv2 cannot decode it, not flagged"))
    elif not err and not jc.equals_golden(golden, name, got):
        bad.append((name, "unflagged, differs from cv2"))


def test_every_case_one_file_per_call(golden, host):
    bad = []
    for name in ACCEPTED:
        (got,), (err,) = device_decode([golden["jpg_" + name]])
        check(golden, host, name, got, err, bad)
    assert not bad, bad


def test_mixed_batch_with_the_cv2_fixtures(golden, golden_dir, host):
    base = np.load(os.path.join(golden_dir, "jpeg_cases.npz"))
    files = [("f", n) for n in ACCEPTED] + [("c", c[0]) for c in jc.CASES]
    np.random.RandomState(5).shuffle(files)
    got, errs = device_decode([(golden if k == "f" else base)["jpg_" + n] for k, n in files])
    bad = []
    for (kind, name), g, e in zip(files, got, errs):
        if kind == "f":
            check(golden, host, name, g, e, bad)
        elif e or not jc.equals_golden(base, name, g):
            bad.append((name, e))
    assert not bad, bad


def test_decode_jpeg_names_the_flags_of_a_damaged_file(golden):
    good = golden["jpg_hdr_plain"]
    with pytest.raises(eng.Yfv2Error, match=r"1 of 2 files failed to decode: b\.jpg: restart markers out of sequence"):
        eng.decode_jpeg([good, golden["jpg_rst_renumbered_5_plus1"]], "cuda", names=["a.jpg", "b.jpg"])
    with pytest.raises(eng.Yfv2Error, match=r"b\.jpg: entropy-coded data ran out"):
        eng.decode_jpeg([good, golden["jpg_hdr_no_eoi"]], "cuda", names=["a.jpg", "b.jpg"])

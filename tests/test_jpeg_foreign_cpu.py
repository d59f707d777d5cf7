"""JPEG files from other encoders, rewritten headers, hand-built entropy data, EXIF variants and damaged scans
(tests/jpeg_foreign_cases.py) through the host parser and the address-sanitised CPU build of the decode (tests/jpeg_harness.cu),
against what cv2.imdecode made of each.  The contract: a file the decoder accepts and does not flag is cv2's frame byte for byte;
a file cv2 cannot decode is refused or flagged; no other file but a damaged scan is flagged; a refused file names why; nothing is
read past a file's end (the harness compiles the parser in with the decode, so AddressSanitizer watches both)."""
import ctypes

import numpy as np
import pytest

import yfv2  # noqa: F401  (registers the package dir)
import jpeg_cases as jc
import jpeg_foreign_cases as fc
from test_jpeg_cpu import harness, run_harness  # noqa: F401  (the harness fixture, built once per module)


@pytest.fixture(scope="module")
def golden(golden_dir):
    import os
    return np.load(os.path.join(golden_dir, "jpeg_foreign.npz"))


def parse_one(buf):
    import yfv2_engine
    L = yfv2_engine.lib()
    info = yfv2_engine.JpegInfo()
    sz = ctypes.c_size_t()
    rc = L.yfv2_jpeg_parse(buf.ctypes.data, (ctypes.c_longlong * 2)(0, buf.size), 1, ctypes.byref(info), None, 0,
                           ctypes.byref(sz), ctypes.byref(sz), ctypes.byref(sz))
    return rc, info


def test_goldens_hold_every_case(golden):
    assert sorted(k[4:] for k in golden.files if k.startswith("jpg_")) == sorted(fc.CASES)
    for name in fc.CASES:
        assert ("none_" + name in golden.files) != ("shape_" + name in golden.files), name
    assert set(fc.DAMAGED) <= set(fc.CASES) and set(fc.REFUSED) <= set(fc.CASES)


def test_parser_accepts_or_refuses_each_case_with_its_reason(golden):
    wrong = []
    for name in fc.CASES:
        rc, info = parse_one(golden["jpg_" + name])
        if name in fc.REFUSED:
            code, reason = fc.REFUSED[name]
            if (rc, info.status) != (code, code) or reason not in info.reason.decode():
                wrong.append((name, rc, info.reason.decode()))
        elif rc != 0:
            wrong.append((name, rc, info.reason.decode()))
        elif "shape_" + name in golden.files and (info.h, info.w, 3) != jc.golden_shape(golden, name):
            wrong.append((name, "size", info.h, info.w))
    assert not wrong, wrong


def test_cpu_build_equals_cv2_unless_flagged(golden, harness):  # noqa: F811
    items = [(n, golden["jpg_" + n]) for n in fc.CASES]
    results, outs = run_harness(harness, items)                       # a read past a file's end fails the harness run
    differ, unflagged_none, flagged_clean, refused = [], [], [], []
    for (name, _), (status, w, h, err), out in zip(items, results, outs):
        if status != 0:
            if name not in fc.REFUSED:
                refused.append(name)
            continue
        if err and name not in fc.DAMAGED and "none_" + name not in golden.files:
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


def test_damaged_cases_include_flagged_and_unflagged_files(golden, harness):  # noqa: F811
    """The damaged scans exercise both sides of the contract: some changes leave a scan that cv2 and the decode still agree on
    (unflagged, equal), others are flagged."""
    items = [(n, golden["jpg_" + n]) for n in fc.DAMAGED]
    results, _ = run_harness(harness, items)
    flagged = {n for (n, _), r in zip(items, results) if r[3]}
    assert flagged and set(fc.DAMAGED) - flagged

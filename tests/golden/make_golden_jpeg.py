"""Generates tests/golden/jpeg_cases.npz: the JPEG files of tests/jpeg_cases.py, encoded by cv2.imencode, and cv2.imdecode(bytes,
IMREAD_COLOR) of each (what cv2.imread returns for the same file: in full up to jpeg_cases.FULL_BYTES, else its SHA-256), plus the files the decoder must refuse.  OpenCV is present where
goldens are generated only, so no test calls cv2.  The versions go to tests/golden/META_jpeg.json.

    python tests/golden/make_golden_jpeg.py [--reference /root/reference]

The reference's img/000139.jpg and img/000004.jpg are copied next to it as data fixtures (their cv2.imread bytes are already in
frames_modelzoo.npz; this script checks that they agree)."""
import argparse
import json
import os
import shutil
import struct
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))


def markers(b):
    """(offset of the FF, marker byte, segment length) of every marker from SOI up to and including the first SOS."""
    out, pos = [], 2
    while pos < len(b):
        assert b[pos] == 0xFF
        m = b[pos + 1]
        n = struct.unpack(">H", b[pos + 2:pos + 4])[0]
        out.append((pos, m, n))
        pos += 2 + n
        if m == 0xDA:
            break
    return out


def find(b, m):
    return next(p for p, mm, _ in markers(b) if mm == m)


def exif_app1(orientation, order):
    """APP1 with a TIFF header in byte order `order` and an IFD0 holding only Orientation (tag 0x0112, SHORT)."""
    e = "<" if order == "II" else ">"
    tiff = order.encode() + struct.pack(e + "HI", 42, 8) + struct.pack(e + "H", 1)
    tiff += struct.pack(e + "HHI", 0x0112, 3, 1) + struct.pack(e + "HH", orientation, 0) + struct.pack(e + "I", 0)
    payload = b"Exif\0\0" + tiff
    return b"\xff\xe1" + struct.pack(">H", len(payload) + 2) + payload


def encode(cv2, case):
    import jpeg_cases as jc
    name, seed, (h, w), s, q, opt, rst, orient, order = case
    img = jc.image(seed, h, w, smooth=(h * w > 1_000_000))
    params = [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_OPTIMIZE, opt, cv2.IMWRITE_JPEG_RST_INTERVAL, rst]
    if s == "grey":
        img = cv2.cvtColor(img, cv2.COLOR_BGR2GRAY)
    else:
        params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, getattr(cv2, "IMWRITE_JPEG_SAMPLING_FACTOR_" + s)]
    ok, buf = cv2.imencode(".jpg", img, params)
    assert ok
    b = buf.tobytes()
    if orient is not None:
        b = b[:2] + exif_app1(orient, order) + b[2:]
    return b


def patch(b, off, val):
    b = bytearray(b)
    b[off] = val
    return bytes(b)


def unsupported(cv2, base):
    """The refused files, from one baseline 4:2:0 file `base`."""
    import jpeg_cases as jc
    sof = find(base, 0xC0)
    sos = find(base, 0xDA)
    img = jc.image(7, 40, 40)
    out = {}
    out["progressive"] = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes()
    out["sof2"] = patch(base, sof + 1, 0xC2)
    out["sof3"] = patch(base, sof + 1, 0xC3)
    out["sof9"] = patch(base, sof + 1, 0xC9)
    out["bits12"] = patch(base, sof + 4, 12)
    out["comp4"] = patch(base, sof + 9, 4)
    out["comp2"] = patch(base, sof + 9, 2)
    eoi = base.rindex(b"\xff\xd9")
    out["two_scans"] = base[:eoi] + base[sos:eoi] + base[eoi:]                      # the scan again after the first one
    app0 = find(base, 0xE0)
    n0 = struct.unpack(">H", base[app0 + 2:app0 + 4])[0]
    adobe = b"\xff\xee" + struct.pack(">H", 14) + b"Adobe" + struct.pack(">HHHB", 100, 0, 0, 0)
    out["adobe_rgb"] = base[:app0] + adobe + base[app0 + 2 + n0:]                   # JFIF APP0 replaced by Adobe, transform 0
    out["sampling_22_21"] = patch(base, sof + 10 + 3 + 1, 0x21)                    # Cb sampled 2x1 under 2x2 luma
    out["png"] = cv2.imencode(".png", img)[1].tobytes()
    out["cut_header"] = base[:sos - 40]
    assert set(out) == {n for n, _, _ in jc.UNSUPPORTED}
    return out


def main():
    import cv2
    import jpeg_cases as jc
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default="/root/reference")
    args = ap.parse_args()
    out = {}
    for case in jc.CASES:
        b = encode(cv2, case)
        out["jpg_" + case[0]] = np.frombuffer(b, np.uint8)
        dec = cv2.imdecode(out["jpg_" + case[0]], cv2.IMREAD_COLOR)
        out["shape_" + case[0]] = np.array(dec.shape, np.int64)
        out["sha_" + case[0]] = jc.digest(dec)
        if dec.nbytes <= jc.FULL_BYTES:
            out["bgr_" + case[0]] = dec
    base = encode(cv2, ("base", 5, (40, 40), "420", 90, 0, 0, None, None))
    for name, b in unsupported(cv2, base).items():
        out["bad_" + name] = np.frombuffer(b, np.uint8)
    big = encode(cv2, ("cut", 6, (64, 96), "420", 95, 0, 0, None, None))
    sos = find(big, 0xDA)
    out["cut_" + jc.TRUNCATED_SCAN] = np.frombuffer(big[:sos + (len(big) - sos) // 2], np.uint8)
    np.savez_compressed(os.path.join(HERE, "jpeg_cases.npz"), **out)
    modelzoo = np.load(os.path.join(HERE, "frames_modelzoo.npz"))
    for stem in ("000139", "000004"):
        dst = os.path.join(HERE, stem + ".jpg")
        shutil.copyfile(os.path.join(args.reference, "img", stem + ".jpg"), dst)
        assert np.array_equal(cv2.imread(dst), modelzoo[stem]), stem
    meta = {"generator": "tests/golden/make_golden_jpeg.py", "opencv": cv2.__version__,
            "libjpeg_turbo": "3.1.2 (OpenCV's bundled build-libjpeg-turbo)", "numpy": np.__version__,
            "cases": len(jc.CASES), "unsupported": len(jc.UNSUPPORTED)}
    with open(os.path.join(HERE, "META_jpeg.json"), "w") as f:
        json.dump(meta, f, indent=1, sort_keys=True)
    print("wrote %d arrays" % len(out))


if __name__ == "__main__":
    main()

"""Writes tests/golden/jpeg_encode_cases.npz: cv2.imencode's bytes for every case of tests/jpeg_encode_cases.py (OpenCV 4.13,
libjpeg-turbo 3.1), the large ones as SHA-256 + length, and cv2.imdecode's frame of the round-trip cases as SHA-256."""
import hashlib
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import jpeg_encode_cases as C  # noqa: E402


def image(c):
    """The BGR (or grey) image cv2 encodes for case c"""
    if c["photo"]:
        f = cv2.imread(os.path.join(HERE, c["photo"]))
    else:
        f = C.frame(c["layout"], c["w"], c["h"], c["kind"], c["seed"])
        code = C.CVT[c["layout"]]
        if c["layout"] == "rgb_chw":
            f = np.ascontiguousarray(f.transpose(1, 2, 0))
        if code:
            f = cv2.cvtColor(f, getattr(cv2, code))
    if c["region"]:
        x0, y0, w, h = c["region"]
        f = np.ascontiguousarray(f[y0:y0 + h, x0:x0 + w])
    return f


def params(c):
    return [cv2.IMWRITE_JPEG_QUALITY, c["quality"], cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
            {"420": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, "422": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
             "444": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444}[c["sampling"]], cv2.IMWRITE_JPEG_RST_INTERVAL, c["restart"]]


def main():
    assert cv2.__version__.startswith("4.13"), cv2.__version__
    out = {}
    for c in C.cases():
        img = image(c)
        b = cv2.imencode(".jpg", img, params(c))[1].tobytes()
        if img.shape[0] * img.shape[1] > C.LARGE:
            out[c["name"] + ".sha"] = np.frombuffer(hashlib.sha256(b).digest(), np.uint8)
            out[c["name"] + ".len"] = np.array(len(b), np.int64)
        else:
            out[c["name"]] = np.frombuffer(b, np.uint8)
        if c["name"] in C.ROUNDTRIP:
            dec = cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)
            out[c["name"] + ".decoded"] = np.frombuffer(hashlib.sha256(dec.tobytes()).digest(), np.uint8)
    np.savez_compressed(os.path.join(HERE, "jpeg_encode_cases.npz"), **out)
    print(len(C.cases()), "cases")


if __name__ == "__main__":
    main()

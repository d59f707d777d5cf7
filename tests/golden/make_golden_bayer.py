"""Generates tests/golden/bayer_cases.npz with the REAL cv2 (OpenCV 4.13, x86 build) on the seeded raw Bayer frames of
tests/bayer_cases.py: cv2.cvtColor(raw, COLOR_Bayer??2BGR / _EA), cropped to the case's window, then cv2.resize INTER_LINEAR;
and cv2.imencode of the converted frame's window and region.  OpenCV is present in the build container only, so no test calls
cv2: they compare against what this script froze.

    python tests/golden/make_golden_bayer.py

For resize case <name>: `<name>_in_sha256` (of the raw frame's bytes, to catch a changed input generator), `<name>_bgr_sha256`
(of cv2's converted window, the image before the resize), `<name>_sha256` (of cv2's [H, W, 3] resize), and `<name>_bgr` /
`<name>_out` themselves when they are at most 4 KB.  For encode case <name>: `<name>.img_sha256` (of the image encoded) and
`<name>.jpg` (cv2.imencode's bytes), or for images larger than 4 KB `<name>.sha` and `<name>.len`.  The script asserts that
tests/bayer_oracle.py gives cv2's converted bytes for every case.  The versions go to tests/golden/META_bayer.json.
"""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (os.path.dirname(os.path.dirname(HERE)), os.path.dirname(HERE)):    # the repository (oracle/) and tests/
    sys.path.insert(0, p)


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def main():
    import cv2
    import bayer_cases as bc
    import bayer_oracle as bo
    assert cv2.__version__.startswith("4.13"), cv2.__version__

    def cv2_bgr(raw, layout):
        return cv2.cvtColor(np.ascontiguousarray(raw), getattr(cv2, bc.CODES[layout]))

    out = {}
    for case in bc.CASES:
        name, layout, _, _, (H, W), _, _ = case
        raw = bc.case_input(case)
        x0, y0, w, h = bc.window_of(case)
        bgr = np.ascontiguousarray(cv2_bgr(raw, layout)[y0:y0 + h, x0:x0 + w])
        assert np.array_equal(bgr, bo.window_bgr(raw, layout, x0, y0, w, h)), name
        dst = cv2.resize(bgr, (W, H), interpolation=cv2.INTER_LINEAR)
        assert dst.shape == (H, W, 3) and dst.dtype == np.uint8
        out[name + "_in_sha256"] = sha(raw)
        out[name + "_bgr_sha256"] = sha(bgr)
        out[name + "_sha256"] = sha(dst)
        if bgr.nbytes <= bc.FULL_BYTES:
            out[name + "_bgr"] = bgr
        if dst.nbytes <= bc.FULL_BYTES:
            out[name + "_out"] = dst
    sampling = {"420": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, "422": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
                "444": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444}
    for c in bc.ENCODE_CASES:
        img = bc.encode_image(c, cv2_bgr)
        assert np.array_equal(img, bc.encode_image(c, bo.to_bgr)), c["name"]
        out[c["name"] + ".img_sha256"] = sha(img)
        b = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, c["quality"], cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                                       sampling[c["sampling"]]])[1].tobytes()
        if img.nbytes > bc.FULL_BYTES:
            out[c["name"] + ".sha"] = np.frombuffer(hashlib.sha256(b).digest(), np.uint8)
            out[c["name"] + ".len"] = np.array(len(b), np.int64)
        else:
            out[c["name"] + ".jpg"] = np.frombuffer(b, np.uint8)
    np.savez_compressed(os.path.join(HERE, "bayer_cases.npz"), **out)
    meta = {"opencv": cv2.__version__, "numpy": np.__version__,
            "bayer_cases": "tests/golden/make_golden_bayer.py: cv2.cvtColor COLOR_Bayer{BG,GB,RG,GR}2BGR and _EA on the seeded "
                           "raw frames of tests/bayer_cases.py, cropped to each case's window, then cv2.resize INTER_LINEAR (x86 "
                           "build); cv2.imencode('.jpg') of the converted windows and regions at the cases' quality and sampling"}
    with open(os.path.join(HERE, "META_bayer.json"), "w") as f:
        json.dump(meta, f)
    print("wrote bayer_cases.npz (cv2 %s)" % cv2.__version__)


if __name__ == "__main__":
    main()

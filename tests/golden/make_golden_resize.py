"""Generates tests/golden/resize_cases.npz with the REAL cv2.resize call of the reference (test.py:35, utils/datasets.py:107:
INTER_LINEAR to (width, height)) on the seeded frames of tests/resize_cases.py, and tests/golden/frames_modelzoo.npz with the
reference's bundled img/000139.jpg and img/000004.jpg as cv2.imread decodes them.  OpenCV is present in the build container only,
and builds for other CPUs may round differently, so no test calls cv2: they compare against what this script froze.

    python tests/golden/make_golden_resize.py [--reference /root/reference]

resize_cases.npz holds per case `<name>_sha256` (SHA-256 of cv2's [H, W, 3] output bytes) and `<name>_in_sha256` (of the resized
window, to catch a changed input generator), plus `<name>_out` (the output itself) when it is at most 48 KB.  The versions and
sources these goldens were made with go to tests/golden/META_resize.json (META.json records the other generators).
"""
import argparse
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

FULL_BYTES = 48 * 1024


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def main():
    import cv2
    import resize_cases as rc
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default="/root/reference")
    args = ap.parse_args()
    out = {}
    for case in rc.CASES:
        name, _, _, _, (H, W) = case
        _, src = rc.case_input(case)
        dst = cv2.resize(src, (W, H), interpolation=cv2.INTER_LINEAR)
        assert dst.shape == (H, W, 3) and dst.dtype == np.uint8
        out[name + "_sha256"] = sha(dst)
        out[name + "_in_sha256"] = sha(src)
        if dst.nbytes <= FULL_BYTES:
            out[name + "_out"] = dst
    np.savez_compressed(os.path.join(HERE, "resize_cases.npz"), **out)
    frames = {}
    for name in rc.MODELZOO_FRAMES:
        frames[name] = cv2.imread(os.path.join(args.reference, "img", name + ".jpg"))
    np.savez_compressed(os.path.join(HERE, "frames_modelzoo.npz"), **frames)
    meta = {"opencv": cv2.__version__, "numpy": np.__version__, "reference_commit": "ac2a5e3",
            "resize_cases": "tests/golden/make_golden_resize.py: cv2.resize INTER_LINEAR (x86 build) on the seeded frames of "
                            "tests/resize_cases.py",
            "frames_modelzoo": "cv2.imread of the reference's img/000139.jpg, img/000004.jpg"}
    with open(os.path.join(HERE, "META_resize.json"), "w") as f:
        json.dump(meta, f)
    print("wrote resize_cases.npz, frames_modelzoo.npz (cv2 %s)" % cv2.__version__)


if __name__ == "__main__":
    main()

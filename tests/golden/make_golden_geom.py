"""Generates tests/golden/geom_cases.npz with the REAL cv2 (OpenCV 4.13, x86 build) for the cases of tests/geom_cases.py: per
output image, load_mosaic's canvas in numpy (or the image alone), cv2.warpAffine(canvas, M[:2], (W, H), borderValue=(114, 114,
114)) or cv2.warpPerspective(canvas, M, (W, H), borderValue=...) INTER_LINEAR, then np.fliplr; and the targets by YOLOv5's own
label lines (tests/geom_oracle.py: yolov5_labels).  OpenCV is present in the build container only, so no test calls cv2: they
compare against what this script froze.

    python tests/golden/make_golden_geom.py

For case <name>: `<name>_M`, `<name>_meta` and `<name>_s` (the draws: matrices, flags and tiles as tests/geom_cases.py packs them,
so the tests do not depend on libm), `<name>_sha256` (of cv2's planar [N, 3, H, W] output), `<name>_out` itself when it is at
most 16 KB, and `<name>_labels` (YOLOv5's targets of the output).  `jpeg_imgs`: the bundled 000004 / 000139 as cv2.imread +
cv2.resize INTER_LINEAR to 96 x 96 gave them.  The script asserts that tests/geom_oracle.py gives cv2's bytes for every case and
that the identity case returns its input.  The versions go to tests/golden/META_geom.json."""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.dirname(HERE), os.path.join(ROOT, "yolo-fastestv2_b200")):
    sys.path.insert(0, p)


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def main():
    import cv2
    import geom_cases as gc
    import geom_oracle as go
    assert cv2.__version__.startswith("4.13"), cv2.__version__
    out = {}
    jpeg = np.stack([cv2.resize(cv2.imread(os.path.join(HERE, f)), (96, 96), interpolation=cv2.INTER_LINEAR) for f in gc.JPEGS])
    out["jpeg_imgs"] = jpeg
    for case in gc.CASES:
        name, N, H, W, seed = case[:5]
        ds = gc.draws(case)
        M, meta, s = gc.pack(ds)
        ds = gc.unpack(M, meta, s)                                   # exactly what the tests read back
        batch = gc.images(name, N, H, W, seed, jpeg)
        hwc = np.ascontiguousarray(batch.transpose(0, 2, 3, 1))
        res = []
        for d in ds:
            cv = go.canvas(hwc, d)
            if d["perspective"]:
                w = cv2.warpPerspective(cv, d["M"], (W, H), flags=cv2.INTER_LINEAR, borderValue=(114, 114, 114))
            else:
                w = cv2.warpAffine(cv, d["M"][:2], (W, H), flags=cv2.INTER_LINEAR, borderValue=(114, 114, 114))
            res.append(np.ascontiguousarray(np.fliplr(w) if d["flip"] else w).transpose(2, 0, 1))
        res = np.stack(res)
        assert np.array_equal(go.augment_planar(batch, ds), res), name
        if name == "identity":
            assert np.array_equal(res, batch)
        out[name + "_M"], out[name + "_meta"], out[name + "_s"] = M, meta, s
        out[name + "_sha256"] = sha(res)
        if res.nbytes <= 16384:
            out[name + "_out"] = res
        out[name + "_labels"] = go.yolov5_labels(gc.targets(N, seed), ds, H, W)
    path = os.path.join(HERE, "geom_cases.npz")
    np.savez_compressed(path, **out)
    meta = {"opencv": cv2.__version__, "numpy": np.__version__,
            "geom_cases": "tests/golden/make_golden_geom.py: numpy load_mosaic canvas, cv2.warpAffine / cv2.warpPerspective "
                          "INTER_LINEAR borderValue (114, 114, 114), np.fliplr (x86 build); YOLOv5's label lines"}
    with open(os.path.join(HERE, "META_geom.json"), "w") as f:
        json.dump(meta, f)
    print("wrote", path, len(gc.CASES), "cases")


if __name__ == "__main__":
    main()

"""Generates tests/golden/aug_hsv_cases.npz with the REAL cv2 (cv2.cvtColor COLOR_BGR2HSV / COLOR_HSV2BGR) and the reference's own
augment_hsv, random_resize and contrast_and_brightness (utils/datasets.py:10-61, imported from the reference checkout; build
container only).  Builds of OpenCV for other CPUs may round differently, so no test calls cv2: they compare against this.

    python tests/golden/make_golden_aug_hsv.py [--reference /root/reference]

Contents ("<case>_sha256" is the SHA-256 of cv2's / the reference's [h, w, 3] output bytes, "<case>_out" the output itself when it
is at most 48 KB; inputs are seeded, see tests/aug_hsv_cases.py):
  bgr2hsv_sha256 / hsv2bgr_sha256 / roundtrip_sha256   cv2 over the 4096 x 4096 image of all 2^24 byte triples (HSV2BGR reads
                                                       the triples as HSV; the round trip is HSV2BGR(BGR2HSV(.)));
  hsv2bgr_col_sha256 / hsv2bgr_w53_sha256              HSV2BGR of the same triples as rows of 1 pixel (all in cv2's scalar
                                                       tail) and of its first 4081 columns as rows of 53 (32 vector + 21 tail);
  hsv_<case>_{u,r,luts}                                augment_hsv with np.random.uniform returning u, r = u * gains + 1, and the
                                                       three LUTs the reference passed to cv2.LUT;
  rr_<case>_{rw,rh}                                    random_resize with random.uniform returning the draws for (rw, rh);
  chain_<seed>_{alpha,beta,rw,rh,r}, chain_<seed>_<i>_sha256
                                                       contrast -> random_resize -> augment_hsv per image after random.seed(seed)
                                                       and np.random.seed(seed), the draws as the reference made them.
The versions go to tests/golden/META_aug_hsv.json."""
import argparse
import hashlib
import json
import os
import random
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (os.path.dirname(os.path.dirname(HERE)), os.path.dirname(HERE)):    # the repository (oracle/) and tests/
    sys.path.insert(0, p)

FULL_BYTES = 48 * 1024


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def put(out, name, img):
    out[name + "_sha256"] = sha(img)
    if img.nbytes <= FULL_BYTES:
        out[name + "_out"] = img


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default="/root/reference")
    args = ap.parse_args()
    sys.path.insert(0, args.reference)
    import cv2
    import utils.datasets as ds
    import aug_hsv_cases as hc
    import aug_hsv_oracle as ho
    cv2.setNumThreads(1)
    out = {}

    cube = ho.all_triples()
    out["bgr2hsv_sha256"] = sha(cv2.cvtColor(cube, cv2.COLOR_BGR2HSV))
    out["hsv2bgr_sha256"] = sha(cv2.cvtColor(cube, cv2.COLOR_HSV2BGR))
    out["roundtrip_sha256"] = sha(cv2.cvtColor(cv2.cvtColor(cube, cv2.COLOR_BGR2HSV), cv2.COLOR_HSV2BGR))
    out["hsv2bgr_col_sha256"] = sha(cv2.cvtColor(cube.reshape(-1, 1, 3), cv2.COLOR_HSV2BGR))    # 1-pixel rows: the scalar tail
    out["hsv2bgr_w53_sha256"] = sha(cv2.cvtColor(cube[:, :4081].reshape(-1, 53, 3), cv2.COLOR_HSV2BGR))

    real_uniform, real_lut = np.random.uniform, cv2.LUT
    for name, img_spec, u in hc.HSV_CASES:
        img = hc.image(*img_spec)
        luts = []
        np.random.uniform = lambda lo, hi, n, u=u: np.array(u, np.float64)
        cv2.LUT = lambda src, lut: (luts.append(np.array(lut)), real_lut(src, lut))[1]
        try:
            dst = ds.augment_hsv(img)
        finally:
            np.random.uniform, cv2.LUT = real_uniform, real_lut
        out["hsv_%s_u" % name] = np.array(u, np.float64)
        out["hsv_%s_r" % name] = np.array(u, np.float64) * list(ho.HSV_GAINS) + 1
        out["hsv_%s_luts" % name] = np.stack(luts)
        put(out, "hsv_" + name, dst)

    real_runiform = random.uniform
    for name, img_spec, (rw, rh) in hc.RESIZE_CASES:
        img = hc.image(*img_spec)
        h, w, _ = img.shape
        uw, uh = (1.0 if rw == w else (rw + 0.5) / w), (1.0 if rh == h else (rh + 0.5) / h)
        assert (int(w * uw), int(h * uh)) == (rw, rh)
        draws = iter([uw, uh])
        random.uniform = lambda lo, hi: next(draws)
        try:
            dst = ds.random_resize(img)
        finally:
            random.uniform = real_runiform
        out["rr_%s_rw" % name], out["rr_%s_rh" % name] = np.int64(rw), np.int64(rh)
        put(out, "rr_" + name, dst)
    for s in hc.RESIZE_SEEDS:                                   # seeded draws, as the reference makes them
        img = hc.image(40 + s, 352, 352)
        random.seed(s)
        dst = ds.random_resize(img)
        g = random.Random(s)
        rw, rh = int(352 * g.uniform(0.8, 1)), int(352 * g.uniform(0.8, 1))
        out["rr_seed%d_rw" % s], out["rr_seed%d_rh" % s] = np.int64(rw), np.int64(rh)
        put(out, "rr_seed%d" % s, dst)

    for s in hc.CHAIN_SEEDS:
        imgs = hc.chain_batch(s)
        random.seed(s)
        np.random.seed(s)
        for i, img in enumerate(imgs):
            put(out, "chain_%d_%d" % (s, i), ds.augment_hsv(ds.random_resize(ds.contrast_and_brightness(img))))
        g, nr = random.Random(s), np.random.RandomState(s)
        d = {"alpha": [], "beta": [], "rw": [], "rh": [], "r": []}
        for img in imgs:
            h, w, _ = img.shape
            d["alpha"].append(g.uniform(0.25, 1.75)); d["beta"].append(g.uniform(0.25, 1.75))
            d["rw"].append(int(w * g.uniform(0.8, 1))); d["rh"].append(int(h * g.uniform(0.8, 1)))
            d["r"].append(nr.uniform(-1, 1, 3) * list(ho.HSV_GAINS) + 1)
        for k, v in d.items():
            out["chain_%d_%s" % (s, k)] = np.array(v)

    np.savez_compressed(os.path.join(HERE, "aug_hsv_cases.npz"), **out)
    meta = {"opencv": cv2.__version__, "numpy": np.__version__, "reference_commit": "ac2a5e3",
            "aug_hsv_cases": "tests/golden/make_golden_aug_hsv.py: cv2.cvtColor COLOR_BGR2HSV / COLOR_HSV2BGR (x86 build) over all "
                             "2^24 byte triples, and the reference's augment_hsv / random_resize / contrast_and_brightness on the "
                             "seeded images of tests/aug_hsv_cases.py"}
    with open(os.path.join(HERE, "META_aug_hsv.json"), "w") as f:
        json.dump(meta, f)
    print("wrote aug_hsv_cases.npz (cv2 %s)" % cv2.__version__)


if __name__ == "__main__":
    main()

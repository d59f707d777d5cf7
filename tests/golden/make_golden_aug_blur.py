"""Generates tests/golden/aug_blur_cases.npz with the REAL cv2 (getRotationMatrix2D, warpAffine, filter2D, normalize) and the
reference's own motion_blur, contrast_and_brightness, random_resize and augment_hsv (utils/datasets.py:10-61, imported from
the reference checkout; build container only).  Builds of OpenCV for other CPUs may round differently, so no test calls cv2:
they compare against this.

    python tests/golden/make_golden_aug_blur.py [--reference /root/reference]

Contents (inputs are seeded, see tests/aug_blur_cases.py; "<case>_sha256" is the SHA-256 of cv2's / the reference's output
bytes, "<case>_out" the output itself when it is at most 48 KB):
  sweep_d<k>_sha256                  the fp32 taps (warpAffine / degree, as filter2D converts them) over aug_blur_cases.SWEEP;
  taps_d<k>_<i>                      the full fp32 taps at FULL_ANGLES[i];
  special_d<k>_taps                  [len(SPECIAL_ANGLES), k, k] taps at the special angles;
  edge1024_d<k>, edge32_d<k>         [n, 2] adjacent angles across which a cvRound'ed 1/1024 term (resp. a 1/32 coordinate)
                                     changes, found by bisection; edge*_d<k>_taps the [n, 2, k, k] taps at both;
  filt_<case>, norm_<case>           cv2.filter2D(img, -1, taps) and cv2.normalize of it (NORM_MINMAX, 0..255) per FILTER_CASES,
                                     plus the constant and striped images (both become constant, so normalize gives zeros);
  blur_<seed>_draws, blur_<seed>_<i> motion_blur per image after random.seed(seed): the draws (randint(1, 2), degree, angle;
                                     degree 0 when no blur) and the output;
  chain_<seed>_{alpha,beta,degree,angle,rw,rh,r}, chain_<seed>_<i>
                                     contrast -> motion_blur -> random_resize -> augment_hsv per image after random.seed(seed) and
                                     np.random.seed(seed), as img_aug with every line enabled; degree 0 is no blur;
  chain_<seed>_calls                 every random / np.random call the reference made, in order: [n, 2] (kind, value) with kind 0
                                     uniform, 1 randint, 2 np.random.uniform (one row per gain).
The versions and the CPU dispatch level go to tests/golden/META_aug_blur.json."""
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
    import aug_blur_cases as bc
    cv2.setNumThreads(1)
    out = {}

    def cv_taps(d, a):
        k = cv2.warpAffine(np.diag(np.ones(d)), cv2.getRotationMatrix2D((d / 2, d / 2), a, 1), (d, d)) / d
        return k.astype(np.float32)                                     # filter2D converts its kernel to fp32

    for d in (2, 3):
        out["sweep_d%d_sha256" % d] = sha(np.stack([cv_taps(d, a) for a in bc.SWEEP]))
        for i, a in enumerate(bc.FULL_ANGLES):
            out["taps_d%d_%d" % (d, i)] = cv_taps(d, a)
        out["special_d%d_taps" % d] = np.stack([cv_taps(d, a) for a in bc.SPECIAL_ANGLES])
        for which, name in ((0, "edge1024"), (1, "edge32")):
            pairs = np.array(bc.find_edges(d, which, 6, 10 * d + which))
            out["%s_d%d" % (name, d)] = pairs
            out["%s_d%d_taps" % (name, d)] = np.stack([[cv_taps(d, a) for a in p] for p in pairs])

    cases = [(n, bc.image(*spec), d, a) for n, spec, d, a in bc.FILTER_CASES]
    cases += [("constant", bc.constant_image(), 3, 27.0), ("striped", bc.striped_image(), 2, 0.0)]
    for name, img, d, a in cases:
        f = cv2.filter2D(img, -1, cv_taps(d, a).astype(np.float64))
        n = f.copy()
        cv2.normalize(n, n, 0, 255, cv2.NORM_MINMAX)
        if name in ("constant", "striped"):
            assert f.min() == f.max() and n.max() == 0, name
        put(out, "filt_" + name, f)
        put(out, "norm_" + name, n)

    real_uniform, real_randint, real_np_uniform = random.uniform, random.randint, np.random.uniform
    calls = []

    def log_uniform(lo, hi):
        v = real_uniform(lo, hi)
        calls.append((0, v))
        return v

    def log_randint(lo, hi):
        v = real_randint(lo, hi)
        calls.append((1, v))
        return v

    def log_np_uniform(lo, hi, n):
        v = real_np_uniform(lo, hi, n)
        calls.extend((2, x) for x in v)
        return v

    for s in bc.BLUR_SEEDS:
        random.seed(s)
        for i, img in enumerate(bc.seeded_batch(s)):
            put(out, "blur_%d_%d" % (s, i), ds.motion_blur(img))
        g, dr = random.Random(s), []
        for _ in range(bc.SEEDED_N):
            dr.append((1, g.randint(2, 3), g.uniform(-360, 360)) if g.randint(1, 2) == 1 else (2, 0, 0.0))
        out["blur_%d_draws" % s] = np.array(dr, np.float64)

    for s in bc.CHAIN_SEEDS:
        random.seed(s)
        np.random.seed(s)
        del calls[:]
        random.uniform, random.randint, np.random.uniform = log_uniform, log_randint, log_np_uniform
        try:
            for i, img in enumerate(bc.seeded_batch(s)):
                put(out, "chain_%d_%d" % (s, i), ds.augment_hsv(ds.random_resize(ds.motion_blur(ds.contrast_and_brightness(img)))))
        finally:
            random.uniform, random.randint, np.random.uniform = real_uniform, real_randint, real_np_uniform
        out["chain_%d_calls" % s] = np.array(calls, np.float64)
        g, nr = random.Random(s), np.random.RandomState(s)
        d = {k: [] for k in ("alpha", "beta", "degree", "angle", "rw", "rh", "r")}
        for _ in range(bc.SEEDED_N):
            d["alpha"].append(g.uniform(0.25, 1.75)); d["beta"].append(g.uniform(0.25, 1.75))
            if g.randint(1, 2) == 1:
                d["degree"].append(g.randint(2, 3)); d["angle"].append(g.uniform(-360, 360))
            else:
                d["degree"].append(0); d["angle"].append(0.0)
            d["rw"].append(int(352 * g.uniform(0.8, 1))); d["rh"].append(int(352 * g.uniform(0.8, 1)))
            d["r"].append(nr.uniform(-1, 1, 3) * [0.0138, 0.678, 0.36] + 1)
        for k, v in d.items():
            out["chain_%d_%s" % (s, k)] = np.array(v)

    np.savez_compressed(os.path.join(HERE, "aug_blur_cases.npz"), **out)
    info = cv2.getBuildInformation()
    line = lambda key: next((l.split(":", 1)[1].strip() for l in info.splitlines() if l.strip().startswith(key)), "?")  # noqa: E731
    meta = {"opencv": cv2.__version__, "numpy": np.__version__, "reference_commit": "ac2a5e3",
            "cpu_baseline": line("Baseline"), "cpu_dispatch": line("Dispatched code"),
            "cpu_runtime": [f for f, i in (("AVX2", 11), ("FMA3", 12), ("AVX_512F", 13), ("AVX512_SKX", 256))   # CV_CPU_* ids
                            if cv2.checkHardwareSupport(i)],
            "aug_blur_cases": "tests/golden/make_golden_aug_blur.py: cv2 getRotationMatrix2D / warpAffine / filter2D / normalize "
                              "(x86 build, one thread) and the reference's motion_blur and img_aug chain on the seeded inputs of "
                              "tests/aug_blur_cases.py"}
    with open(os.path.join(HERE, "META_aug_blur.json"), "w") as f:
        json.dump(meta, f)
    print("wrote aug_blur_cases.npz (cv2 %s)" % cv2.__version__)


if __name__ == "__main__":
    main()

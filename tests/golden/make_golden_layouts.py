"""Generates tests/golden/layout_cases.npz with the REAL cv2.cvtColor (COLOR_RGB2BGR, BGRA2BGR, RGBA2BGR, GRAY2BGR,
YUV2BGR_YUYV / _UYVY / _YVYU) followed by cv2.resize INTER_LINEAR (test.py:35) on the seeded frames of tests/layout_cases.py
and on the bundled images converted to each layout.  OpenCV is present in the build container only, and builds for other CPUs
may round differently, so no test calls cv2: they compare against what this script froze.

    python tests/golden/make_golden_layouts.py

layout_cases.npz holds per case `<name>_sha256` (SHA-256 of cv2's [H, W, 3] output bytes) and `<name>_in_sha256` (of the
frame's bytes, to catch a changed input generator), plus `<name>_out` (the output itself) when it is at most 16 KB.  For the
bundled images (tests/golden/frames_modelzoo.npz) and each layout, `<image>_<layout>_in_sha256` is the SHA-256 of
cv2.cvtColor(img, COLOR_BGR2<LAYOUT>) (planar RGB: the transposed COLOR_BGR2RGB) and `<image>_<layout>_bgr352_sha256` that of
cv2's 352 x 352 BGR resize of the converted frame converted back.  tests/layout_cases.py restates every conversion but the
4:2:2 ones, which this script asserts; cv2's COLOR_BGR2YUV_YUYV is stored as its planes `<image>_yuyv_y` [h, w], `<image>_yuyv_u`
and `<image>_yuyv_v` [h, w/2] (they compress better than the interleaved frame), and the UYVY and YVYU conversions hold the same
samples, which this script also asserts.  The versions go to tests/golden/META_layouts.json.
"""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (os.path.dirname(os.path.dirname(HERE)), os.path.dirname(HERE)):    # the repository (oracle/) and tests/
    sys.path.insert(0, p)

FULL_BYTES = 16 * 1024


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def main():
    import cv2
    import layout_cases as lc
    to_bgr = {"rgb": cv2.COLOR_RGB2BGR, "bgra": cv2.COLOR_BGRA2BGR, "rgba": cv2.COLOR_RGBA2BGR, "gray": cv2.COLOR_GRAY2BGR,
              "rgb_chw": cv2.COLOR_RGB2BGR, "yuyv": cv2.COLOR_YUV2BGR_YUYV, "uyvy": cv2.COLOR_YUV2BGR_UYVY,
              "yvyu": cv2.COLOR_YUV2BGR_YVYU}
    from_bgr = {"rgb": cv2.COLOR_BGR2RGB, "bgra": cv2.COLOR_BGR2BGRA, "rgba": cv2.COLOR_BGR2RGBA, "gray": cv2.COLOR_BGR2GRAY,
                "rgb_chw": cv2.COLOR_BGR2RGB, "yuyv": cv2.COLOR_BGR2YUV_YUYV, "uyvy": cv2.COLOR_BGR2YUV_UYVY,
                "yvyu": cv2.COLOR_BGR2YUV_YVYU}

    def cv2_bgr(frame, layout):
        frame = np.ascontiguousarray(frame.transpose(1, 2, 0) if layout == "rgb_chw" else frame)
        return cv2.cvtColor(frame, to_bgr[layout])

    out = {}
    for case in lc.CASES:
        name, layout, _, (h, w), (H, W), _ = case
        frame = lc.case_input(case)
        bgr = cv2_bgr(frame, layout)
        assert bgr.shape == (h, w, 3), (name, bgr.shape)
        dst = cv2.resize(bgr, (W, H), interpolation=cv2.INTER_LINEAR)
        assert dst.shape == (H, W, 3) and dst.dtype == np.uint8
        out[name + "_sha256"] = sha(dst)
        out[name + "_in_sha256"] = sha(frame)
        if dst.nbytes <= FULL_BYTES:
            out[name + "_out"] = dst
    frames = np.load(os.path.join(HERE, "frames_modelzoo.npz"))
    for img in lc.MODELZOO_FRAMES:
        results = {}
        for layout in lc.LAYOUTS:
            conv = cv2.cvtColor(frames[img], from_bgr[layout])
            if layout == "rgb_chw":
                conv = np.ascontiguousarray(conv.transpose(2, 0, 1))
            results[layout] = cv2.resize(cv2_bgr(conv, layout), (352, 352), interpolation=cv2.INTER_LINEAR)
            out["%s_%s_in_sha256" % (img, layout)] = sha(conv)
            out["%s_%s_bgr352_sha256" % (img, layout)] = sha(results[layout])
            if layout == "yuyv":
                mp = conv.reshape(conv.shape[0], -1, 4)
                out[img + "_yuyv_y"] = np.ascontiguousarray(conv[..., 0])
                out[img + "_yuyv_u"], out[img + "_yuyv_v"] = np.ascontiguousarray(mp[..., 1]), np.ascontiguousarray(mp[..., 3])
            assert np.array_equal(conv, lc.bundled(out, frames, img, layout)), (img, layout)
        assert all(np.array_equal(results[k], results["yuyv"]) for k in lc.YUV422), img
    np.savez_compressed(os.path.join(HERE, "layout_cases.npz"), **out)
    meta = {"opencv": cv2.__version__, "numpy": np.__version__, "reference_commit": "ac2a5e3",
            "layout_cases": "tests/golden/make_golden_layouts.py: cv2.cvtColor COLOR_{RGB,BGRA,RGBA,GRAY}2BGR / "
                            "COLOR_YUV2BGR_{YUYV,UYVY,YVYU} then cv2.resize INTER_LINEAR (x86 build) on the seeded frames of "
                            "tests/layout_cases.py",
            "modelzoo_layouts": "cv2.cvtColor(COLOR_BGR2{RGB,BGRA,RGBA,GRAY,YUV_YUYV,YUV_UYVY,YUV_YVYU}) of the frames in "
                                "tests/golden/frames_modelzoo.npz, and cv2's 352x352 BGR resize of their conversion back to BGR"}
    with open(os.path.join(HERE, "META_layouts.json"), "w") as f:
        json.dump(meta, f)
    print("wrote layout_cases.npz (cv2 %s)" % cv2.__version__)


if __name__ == "__main__":
    main()

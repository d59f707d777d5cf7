"""Generates tests/golden/yuv_cases.npz with the REAL cv2.cvtColor / cv2.cvtColorTwoPlane (COLOR_YUV2BGR_NV12 / _NV21 / _I420 /
_YV12) followed by cv2.resize INTER_LINEAR (test.py:35) on the seeded frames of tests/yuv_cases.py, the 64 colour-cube frames, and
the bundled images converted to I420.  OpenCV is present in the build container only, and builds for other CPUs may round
differently, so no test calls cv2: they compare against what this script froze.

    python tests/golden/make_golden_yuv.py

yuv_cases.npz holds per case `<name>_sha256` (SHA-256 of cv2's [H, W, 3] output bytes) and `<name>_in_sha256` (of the frame's Y,
U and V window bytes, to catch a changed input generator), plus `<name>_out` (the output itself) when it is at most 48 KB;
`cube_<k>_sha256` for the colour-cube frames (NV12, identity size); `<image>_i420` (cv2.cvtColor(img, COLOR_BGR2YUV_I420) of
the decoded bundled image, tests/golden/frames_modelzoo.npz) and `<image>_bgr352` (cv2's 352 x 352 BGR result of it).  The
versions go to tests/golden/META_yuv.json.
"""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (os.path.dirname(os.path.dirname(HERE)), os.path.dirname(HERE)):    # the repository (oracle/) and tests/
    sys.path.insert(0, p)

FULL_BYTES = 48 * 1024


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def planes_sha(planes):
    return sha(np.concatenate([np.ascontiguousarray(p).reshape(-1) for p in planes]))


def main():
    import cv2
    import yuv_cases as yc
    import yuv_oracle as yo
    to_bgr = {"nv12": cv2.COLOR_YUV2BGR_NV12, "nv21": cv2.COLOR_YUV2BGR_NV21, "i420": cv2.COLOR_YUV2BGR_I420,
              "yv12": cv2.COLOR_YUV2BGR_YV12}
    out = {}
    for case in yc.CASES:
        name, layout, _, (h, w), (H, W), _ = case
        frame = yc.case_input(case)
        if isinstance(frame, tuple) and layout in ("nv12", "nv21"):
            y, uv = frame
            bgr = cv2.cvtColorTwoPlane(y, uv.reshape(h // 2, w // 2, 2), to_bgr[layout])
        else:
            bgr = cv2.cvtColor(frame if not isinstance(frame, tuple) else yc.single_buffer(frame, layout), to_bgr[layout])
        assert bgr.shape == (h, w, 3)
        dst = cv2.resize(bgr, (W, H), interpolation=cv2.INTER_LINEAR)
        assert dst.shape == (H, W, 3) and dst.dtype == np.uint8
        out[name + "_sha256"] = sha(dst)
        out[name + "_in_sha256"] = planes_sha(yo.split(frame, layout))
        if dst.nbytes <= FULL_BYTES:
            out[name + "_out"] = dst
    for k in range(yc.CUBE_FRAMES):
        buf = yc.cube_frame(k)
        dst = cv2.resize(cv2.cvtColor(buf, cv2.COLOR_YUV2BGR_NV12), (512, 512), interpolation=cv2.INTER_LINEAR)
        out["cube_%02d_sha256" % k] = sha(dst)
    frames = np.load(os.path.join(HERE, "frames_modelzoo.npz"))
    for name in yc.MODELZOO_FRAMES:
        i420 = cv2.cvtColor(frames[name], cv2.COLOR_BGR2YUV_I420)
        out[name + "_i420"] = i420
        out[name + "_bgr352"] = cv2.resize(cv2.cvtColor(i420, cv2.COLOR_YUV2BGR_I420), (352, 352), interpolation=cv2.INTER_LINEAR)
    np.savez_compressed(os.path.join(HERE, "yuv_cases.npz"), **out)
    meta = {"opencv": cv2.__version__, "numpy": np.__version__, "reference_commit": "ac2a5e3",
            "yuv_cases": "tests/golden/make_golden_yuv.py: cv2.cvtColor / cv2.cvtColorTwoPlane COLOR_YUV2BGR_{NV12,NV21,I420,YV12} "
                         "then cv2.resize INTER_LINEAR (x86 build) on the seeded frames and the colour cube of tests/yuv_cases.py",
            "modelzoo_i420": "cv2.cvtColor(COLOR_BGR2YUV_I420) of the frames in tests/golden/frames_modelzoo.npz, and cv2's 352x352 "
                             "BGR resize of their COLOR_YUV2BGR_I420 conversion"}
    with open(os.path.join(HERE, "META_yuv.json"), "w") as f:
        json.dump(meta, f)
    print("wrote yuv_cases.npz (cv2 %s)" % cv2.__version__)


if __name__ == "__main__":
    main()

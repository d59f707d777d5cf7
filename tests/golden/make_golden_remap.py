"""Generates tests/golden/remap_cases.npz with the REAL cv2 (OpenCV 4.13, x86 build) on the seeded frames and maps of
tests/remap_cases.py: cv2.cvtColor(frame, COLOR_<LAYOUT>2BGR) (cropped to the inner window), cv2.remap(img, map1, map2,
INTER_LINEAR) in the case's map form, cropped to the view's window, then cv2.resize INTER_LINEAR; and cv2.convertMaps of the
edge values.  OpenCV is present in the build container only, so no test calls cv2: they compare against what this script froze.

    python tests/golden/make_golden_remap.py

For case <name>: `<name>_in_sha256` (of the frame's bytes), `<name>_maps_sha256` (of the fixed maps cv2 remaps with:
cv2.convertMaps of float maps, or the fixed maps), `<name>_remap_sha256` (of cv2.remap's window, the image before the resize)
and `<name>_sha256` (of cv2's [H, W, 3] resize), with `<name>_remap` / `<name>_out` themselves when they are at most 4 KB; a
cv2fixed case also stores cv2.initUndistortRectifyMap(..., CV_16SC2)'s maps as `<name>_map1`, `<name>_map2`.  `edge_map1`,
`edge_map2`: cv2.convertMaps(EDGE_VALUES, 0, CV_16SC2).  For encode case k: `enc<k>.sha` and `enc<k>.len` of cv2.imencode of
the case's remapped window (or its region).  The script asserts that tests/remap_oracle.py gives cv2's bytes for
every case.  The versions go to tests/golden/META_remap.json.
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
    import remap_cases as rc
    import remap_oracle as ro
    assert cv2.__version__.startswith("4.13"), cv2.__version__

    def cv2_bgr(frame, layout):
        if layout == "bgr":
            return frame
        if layout == "rgb_chw":
            frame = frame.transpose(1, 2, 0)
        return cv2.cvtColor(np.ascontiguousarray(frame), getattr(cv2, rc.CODES[layout]))

    out, rems = {}, {}
    for c in rc.CASES:
        name, layout = c["name"], c["layout"]
        W, H = c["target"]
        frame = rc.case_frame(c)
        img = cv2_bgr(frame, layout)
        if c["inner"]:
            x0, y0, w, h = c["inner"]
            img = img[y0:y0 + h, x0:x0 + w]
        img = np.ascontiguousarray(img)
        assert np.array_equal(img, ro.inner_bgr(frame, layout, c["inner"])), name
        if c["map"][0] == "cv2fixed":
            w, h = rc.inner_size(c)
            m1, m2 = cv2.initUndistortRectifyMap(rc.camera(w, h), np.array(rc.D5), None, rc.camera(w, h), (w, h), cv2.CV_16SC2)
            out[name + "_map1"], out[name + "_map2"] = m1, m2
            golden = out
        else:
            golden = None
        m1, m2 = rc.case_maps(c, golden)
        if c["form"] == "convert":                                 # the fixed maps cv2 itself makes of the float maps
            mx, my = rc.float_maps(c["map"][0], c["map"][1], c["map"][2], *rc.inner_size(c), c["seed"])
            m1, m2 = cv2.convertMaps(mx, my, cv2.CV_16SC2)
        rem = cv2.remap(img, m1, m2, cv2.INTER_LINEAR)
        f1, f2 = (m1, m2) if m1.dtype == np.int16 else cv2.convertMaps(m1, m2, cv2.CV_16SC2)
        assert np.array_equal(f1, rc.fixed_maps(c, golden)[0]) and np.array_equal(f2, rc.fixed_maps(c, golden)[1]), name
        x0, y0, w, h = rc.view_window(c)
        rem = np.ascontiguousarray(rem[y0:y0 + h, x0:x0 + w])
        assert np.array_equal(rem, ro.remap_window(img, f1, f2, (x0, y0, w, h))), name
        dst = cv2.resize(rem, (W, H), interpolation=cv2.INTER_LINEAR)
        assert np.array_equal(dst, ro.resize_planar(img, f1, f2, (x0, y0, w, h), W, H).transpose(1, 2, 0)), name
        rems[name] = rem
        out[name + "_in_sha256"] = sha(frame)
        out[name + "_maps_sha256"] = sha(np.concatenate([f1.reshape(-1).view(np.uint8), f2.reshape(-1).view(np.uint8)]))
        out[name + "_remap_sha256"] = sha(rem)
        out[name + "_sha256"] = sha(dst)
        if rem.nbytes <= rc.FULL_BYTES:
            out[name + "_remap"] = rem
        if dst.nbytes <= rc.FULL_BYTES:
            out[name + "_out"] = dst
    sampling = {"420": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, "422": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
                "444": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444}
    for k, (name, q, s, region) in enumerate(rc.ENCODE_CASES):
        img = rems[name]
        if region is not None:
            x0, y0, w, h = region
            img = np.ascontiguousarray(img[y0:y0 + h, x0:x0 + w])
        b = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, sampling[s]])[1].tobytes()
        out["enc%d.sha" % k] = np.frombuffer(hashlib.sha256(b).digest(), np.uint8)
        out["enc%d.len" % k] = np.array(len(b), np.int64)
    e1, e2 = cv2.convertMaps(rc.EDGE_VALUES[None], np.zeros_like(rc.EDGE_VALUES)[None], cv2.CV_16SC2)
    out["edge_map1"], out["edge_map2"] = e1, e2
    np.savez_compressed(os.path.join(HERE, "remap_cases.npz"), **out)
    meta = {"opencv": cv2.__version__, "numpy": np.__version__,
            "remap_cases": "tests/golden/make_golden_remap.py: cv2.cvtColor of the seeded frames of tests/remap_cases.py, "
                           "cv2.remap INTER_LINEAR (BORDER_CONSTANT 0) through the cases' float, convertMaps and CV_16SC2 maps, "
                           "cropped to each view's window, then cv2.resize INTER_LINEAR (x86 build); cv2.convertMaps of the edge "
                           "values"}
    with open(os.path.join(HERE, "META_remap.json"), "w") as f:
        json.dump(meta, f)
    print("wrote remap_cases.npz (cv2 %s), %d cases" % (cv2.__version__, len(rc.CASES)))


if __name__ == "__main__":
    main()

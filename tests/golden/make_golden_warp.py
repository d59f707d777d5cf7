"""Generates tests/golden/warp_cases.npz with the REAL cv2 (OpenCV 4.13, x86 build) on the seeded frames and matrices of
tests/warp_cases.py: cv2.cvtColor(frame, COLOR_<LAYOUT>2BGR) (cropped to the inner window), cv2.warpAffine (2x3 M) or
cv2.warpPerspective (3x3 M) INTER_LINEAR with the default BORDER_CONSTANT 0 (| WARP_INVERSE_MAP for inverse cases), cropped to
the view's window, then cv2.resize INTER_LINEAR; cv2.invert(M, DECOMP_LU) of warp_cases.inv_matrices(); and cv2.imencode of a
few warped windows.  OpenCV is present in the build container only, so no test calls cv2: they compare against what this script
froze.

    python tests/golden/make_golden_warp.py

For case <name>: `<name>_M` (the matrix, for the cases whose matrix comes from cos, sin or a solver), `<name>_in_sha256` (of the
frame's bytes), `<name>_warp_sha256` (of cv2's warped window, the image before the resize) and `<name>_sha256` (of cv2's
[H, W, 3] resize), with `<name>_warp` / `<name>_out` themselves when they are at most 4 KB.  `inv_ok` (cv2.invert's return for
each matrix), `inv_sha256` (of all its float64 results) and `inv_head` (the first 64 results).  For encode case k: `enc<k>.sha`
and `enc<k>.len`.  The script asserts that tests/warp_oracle.py gives cv2's bytes for every case and cv2.invert's bits for every
matrix, that each exact rotation equals cv2.rotate, and that each affine case warped through the oracle's inverse with
WARP_INVERSE_MAP gives the same bytes.  The versions go to tests/golden/META_warp.json.
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
    import remap_oracle as ro
    import warp_cases as wc
    import warp_oracle as wo
    assert cv2.__version__.startswith("4.13"), cv2.__version__

    def cv2_bgr(frame, layout):
        if layout == "bgr":
            return frame
        if layout == "rgb_chw":
            frame = frame.transpose(1, 2, 0)
        return cv2.cvtColor(np.ascontiguousarray(frame), getattr(cv2, wc.CODES[layout]))

    def cv2_warp(img, M, dsize, inverse):
        fn = cv2.warpPerspective if M.shape == (3, 3) else cv2.warpAffine
        return fn(img, M, tuple(dsize), flags=cv2.INTER_LINEAR | (cv2.WARP_INVERSE_MAP if inverse else 0))

    out, warps = {}, {}
    for c in wc.CASES:
        name, layout = c["name"], c["layout"]
        W, H = c["target"]
        M = c["M"]
        if name in wc.FROM_GOLDEN:
            out[name + "_M"] = M
        frame = wc.case_frame(c)
        img = cv2_bgr(frame, layout)
        if c["inner"]:
            x0, y0, w, h = c["inner"]
            img = img[y0:y0 + h, x0:x0 + w]
        img = np.ascontiguousarray(img)
        assert np.array_equal(img, ro.inner_bgr(frame, layout, c["inner"])), name
        full = cv2_warp(img, M, c["dsize"], c["inverse"])
        if c["rotate"]:
            assert np.array_equal(full, cv2.rotate(img, getattr(cv2, c["rotate"]))), name
        if M.shape == (2, 3) and not c["inverse"]:
            assert np.array_equal(full, cv2_warp(img, wo.invert_affine(M)[:6].reshape(2, 3), c["dsize"], True)), name
        x0, y0, w, h = wc.view_window(c)
        warp = np.ascontiguousarray(full[y0:y0 + h, x0:x0 + w])
        assert np.array_equal(warp, wo.warp_window(img, M, c["dsize"], (x0, y0, w, h), c["inverse"])), name
        dst = cv2.resize(warp, (W, H), interpolation=cv2.INTER_LINEAR)
        assert np.array_equal(dst, wo.resize_planar(img, M, c["dsize"], (x0, y0, w, h), W, H, c["inverse"]).transpose(1, 2, 0))
        warps[name] = warp
        out[name + "_in_sha256"] = sha(frame)
        out[name + "_warp_sha256"] = sha(warp)
        out[name + "_sha256"] = sha(dst)
        if warp.nbytes <= wc.FULL_BYTES:
            out[name + "_warp"] = warp
        if dst.nbytes <= wc.FULL_BYTES:
            out[name + "_out"] = dst
    horizon = [c for c in wc.CASES if c["name"] == "bgr_horizon_row"][0]
    assert (warps["bgr_horizon_row"][64] == ro.inner_bgr(wc.case_frame(horizon), "bgr")[0, 0]).all()
    sampling = {"420": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, "422": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
                "444": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444}
    for k, (name, q, s, region) in enumerate(wc.ENCODE_CASES):
        img = warps[name]
        if region is not None:
            x0, y0, w, h = region
            img = np.ascontiguousarray(img[y0:y0 + h, x0:x0 + w])
        b = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, sampling[s]])[1].tobytes()
        out["enc%d.sha" % k] = np.frombuffer(hashlib.sha256(b).digest(), np.uint8)
        out["enc%d.len" % k] = np.array(len(b), np.int64)
    mats = wc.inv_matrices()
    oks, invs = [], []
    for m in mats:
        ok, inv = cv2.invert(m, flags=cv2.DECOMP_LU)
        ok2, inv2 = wo.invert_perspective(m)
        assert bool(ok) == ok2 and np.array_equal(inv.reshape(-1), inv2), m
        oks.append(bool(ok))
        invs.append(inv)
    invs = np.array(invs, np.float64)
    assert 0 < sum(oks) < len(oks)
    out["inv_ok"] = np.array(oks)
    out["inv_sha256"] = sha(invs)
    out["inv_head"] = invs[:64]
    np.savez_compressed(os.path.join(HERE, "warp_cases.npz"), **out)
    meta = {"opencv": cv2.__version__, "numpy": np.__version__,
            "warp_cases": "tests/golden/make_golden_warp.py: cv2.cvtColor of the seeded frames of tests/warp_cases.py, "
                          "cv2.warpAffine / cv2.warpPerspective INTER_LINEAR (BORDER_CONSTANT 0, with and without "
                          "WARP_INVERSE_MAP), cropped to each view's window, then cv2.resize INTER_LINEAR (x86 build); "
                          "cv2.invert DECOMP_LU of warp_cases.inv_matrices(); cv2.imencode of warped windows"}
    with open(os.path.join(HERE, "META_warp.json"), "w") as f:
        json.dump(meta, f)
    print("wrote warp_cases.npz (cv2 %s), %d cases, %d matrices" % (cv2.__version__, len(wc.CASES), len(mats)))


if __name__ == "__main__":
    main()

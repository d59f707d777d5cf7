"""Golden vectors for the deploy post-process's parameter space (tests/ncnn_space.py): outputs of the REFERENCE's own C++
(sample/ncnn/src/yolo-fastestv2.cpp predHandle + nmsHandle, compiled in place by `make -C oracle ref` against stub ncnn / OpenCV
headers, as make_golden_ncnn.py does) on every case whose order the reference fixes: no score shared by two passing candidates,
or at most 16 passing candidates (libstdc++'s std::sort is a stable insertion sort up to 16 elements).  The other cases are
compared with oracle/ncnn_post.c only.

Run where the reference is mounted:  python tests/golden/make_golden_ncnn_space.py
Inputs are stored with the outputs, so the fixture does not depend on the host's exp().  Re-running reproduces the file byte for
byte: fixed seeds, and the archive is written with fixed member order and timestamps.
"""
import ctypes
import json
import os
import platform
import subprocess
import sys
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import ncnn_space as ns  # noqa: E402

subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "ref"], check=True, capture_output=True)
ref = ctypes.CDLL(os.path.join(ROOT, "oracle", "_ref", "libncnn_post_ref.so"))
ref.ncnn_ref_detect.restype = ctypes.c_int
ref.ncnn_ref_detect.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
ref.ncnn_ref_configure.restype = None
ref.ncnn_ref_configure.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_void_p]


def run_ref(c):
    o2, o3 = np.ascontiguousarray(c["out2"]), np.ascontiguousarray(c["out3"])
    anc = np.ascontiguousarray(c["anchors"], np.float32)
    ref.ncnn_ref_configure(c["A"], c["C"], c["W"], c["H"], c["nms"], anc.ctypes.data)
    cap = max(ns.slots(c["A"], c["H"], c["W"]), 1)
    boxes = np.zeros((cap, 4), np.int32); scores = np.zeros(cap, np.float32); cates = np.zeros(cap, np.int32)
    n = ref.ncnn_ref_detect(o2.ctypes.data, o2.shape[0], o2.shape[1], o3.ctypes.data, o3.shape[0], o3.shape[1], o2.shape[2],
                            c["src"][0], c["src"][1], c["thresh"], cap, boxes.ctypes.data, scores.ctypes.data, cates.ctypes.data)
    return boxes[:n].copy(), scores[:n].copy(), cates[:n].copy()


out, names, skipped = {}, [], []
for c in ns.cases_all() + ns.limit_cases():
    ns.check(c)
    if not ns.golden_ok(c):
        skipped.append(c["name"])
        continue
    b, s, k = run_ref(c)
    print("%-22s passed %5d kept %5d" % (c["name"], int(ns.candidates(c)["passed"].sum()), len(s)))
    n = c["name"]
    names.append(n)
    out[n + "_out2"] = c["out2"]; out[n + "_out3"] = c["out3"]
    out[n + "_params"] = np.array([c["A"], c["C"], c["W"], c["H"], c["src"][0], c["src"][1]], np.int64)
    out[n + "_fparams"] = np.array([c["thresh"], c["nms"]], np.float32)
    out[n + "_anchors"] = np.asarray(c["anchors"], np.float32)
    out[n + "_boxes"] = b; out[n + "_scores"] = s; out[n + "_cates"] = k
out["names"] = np.array(names)
path = os.path.join(HERE, "ncnn_space.npz")
with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:          # np.savez_compressed stamps members with the current time
    for key, arr in out.items():
        info = zipfile.ZipInfo(key + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
        info.compress_type = zipfile.ZIP_DEFLATED
        with z.open(info, "w", force_zip64=True) as f:
            np.lib.format.write_array(f, np.asanyarray(arr), allow_pickle=False)
print("wrote", path, os.path.getsize(path), "bytes;", len(names), "cases;", "oracle only:", skipped)
meta = {
    "file": "tests/golden/ncnn_space.npz",
    "generator": "tests/golden/make_golden_ncnn_space.py",
    "reference": "sample/ncnn/src/yolo-fastestv2.cpp (yoloFastestv2::detection: predHandle + nmsHandle), compiled unmodified by "
                 "`make -C oracle ref` (g++ -O2 -ffp-contract=off, stub ncnn / OpenCV headers of oracle/ncnn_shim/)",
    "host": "%s %s, %s" % (platform.machine(), platform.system(), subprocess.run(["g++", "--version"], capture_output=True,
                                                                                 text=True).stdout.splitlines()[0]),
    "cases": names,
    "oracle_only": skipped,
    "selection": "cases whose passing candidates share no score, or number at most 16 (std::sort is a stable insertion sort "
                 "there); the others have an order among ties the reference leaves to introsort",
    "inputs": "tests/ncnn_space.py builders (seeded numpy), stored with the outputs",
    "numpy": np.__version__,
    "reference_commit": "ac2a5e3",
}
with open(os.path.join(HERE, "META_ncnn_space.json"), "w") as f:
    json.dump(meta, f, indent=1)
    f.write("\n")

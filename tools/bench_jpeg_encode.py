"""Device time of the JPEG encode (yfv2_jpeg_encode) per call, split by stage, against cv2.imencode in host threads.
  python tools/bench_jpeg_encode.py [--n 256] [--reps 20] [--out FILE]
Cases: N full-HD BGR frames, N full-HD NV12 frames and N full-HD raw Bayer frames (RGGB, "bayer_bg", bilinear and edge-aware: the
mosaic of the BGR frames) at quality 95, 4:2:0 (smooth seeded content, so the files are photo-sized), and N detection crops of
assorted sizes from the BGR frames.  Each stage is timed with CUDA events over `reps` calls, the stages
alternated within every repetition; medians are printed with the card's name, power limit and SM clock limit."""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "yolo-fastestv2_b200"))
import yfv2_engine as eng  # noqa: E402
import ctypes  # noqa: E402


def smooth_frames(n, h, w, seed):
    rng = np.random.RandomState(seed)
    out = []
    for _ in range(4):
        small = torch.from_numpy(rng.randint(0, 256, (1, 3, h // 24, w // 24)).astype(np.float32))
        big = torch.nn.functional.interpolate(small, size=(h, w), mode="bicubic", align_corners=False)
        big = big + torch.from_numpy(rng.normal(0, 6, (1, 3, h, w)).astype(np.float32))
        out.append(big.clamp(0, 255).to(torch.uint8)[0].permute(1, 2, 0).contiguous().numpy())
    return [out[i % 4] for i in range(n)]


class Call:
    """One planned encode whose stages can be launched separately"""

    def __init__(self, frames, layout, regions=None):
        self.keep = []
        self.n = len(regions) if regions else len(frames)
        srcs = (eng.JpegEncSrc * self.n)()
        descs = {}
        regions = regions or [(i, 0, 0, None, None) for i in range(len(frames))]
        params = (ctypes.c_int * 6)(1, 95, 7, 0x221111, 4, 0)
        for k, r in enumerate(regions):
            i = r[0]
            if i not in descs:
                f = eng._check_frame(frames[i], layout, i, "bench_jpeg_encode")
                descs[i] = eng._describe(f, layout, torch.device("cuda"), self.keep)
            srcs[k] = descs[i]
            d = srcs[k]
            d.x0, d.y0 = r[1], r[2]
            if r[3] is not None:
                d.w, d.h = r[3], r[4]
            d.params, d.nparams = ctypes.cast(params, ctypes.POINTER(ctypes.c_int)), 6
        self.params = params
        L = eng.lib()
        mb, wb, ab = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_size_t()
        assert L.yfv2_jpeg_encode_plan(srcs, self.n, None, 0, ctypes.byref(mb), ctypes.byref(wb), None, ctypes.byref(ab)) == 0
        self.meta = torch.empty(mb.value, dtype=torch.uint8)
        assert L.yfv2_jpeg_encode_plan(srcs, self.n, ctypes.c_void_p(self.meta.data_ptr()), mb.value, ctypes.byref(mb),
                                       ctypes.byref(wb), None, ctypes.byref(ab)) == 0
        self.meta_dev = self.meta.cuda()
        self.ws = torch.empty(wb.value, dtype=torch.uint8, device="cuda")
        self.arena = torch.empty(ab.value, dtype=torch.uint8, device="cuda")
        self.lengths = torch.empty(self.n, dtype=torch.int64, device="cuda")
        self.sizes = (mb.value, wb.value, ab.value)

    def run(self, phases):
        rc = eng.lib().yfv2_jpeg_encode(ctypes.c_void_p(self.meta.data_ptr()), ctypes.c_void_p(self.meta_dev.data_ptr()), self.sizes[0],
                                        ctypes.c_void_p(self.ws.data_ptr()), self.sizes[1], ctypes.c_void_p(self.arena.data_ptr()),
                                        self.sizes[2], ctypes.c_void_p(self.lengths.data_ptr()), phases,
                                        ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == 0, eng.lib().yfv2_last_error()


STAGES = [("transform", 1), ("scan", 2), ("pack", 4), ("stuff", 8), ("all", 15)]


def time_call(call, reps):
    call.run(15)
    torch.cuda.synchronize()
    t = {k: [] for k, _ in STAGES}
    for _ in range(reps):
        for name, ph in STAGES:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            call.run(ph)
            b.record()
            b.synchronize()
            t[name].append(a.elapsed_time(b))
    return {k: float(np.median(v)) for k, v in t.items()}


def host_cv2(images, threads=8, reps=3):
    import cv2
    cv2.setNumThreads(1)
    best = []
    for _ in range(reps):
        t0 = time.perf_counter()
        with ThreadPoolExecutor(threads) as ex:
            list(ex.map(lambda im: cv2.imencode(".jpg", im, [cv2.IMWRITE_JPEG_QUALITY, 95]), images))
        best.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(best))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=256)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_jpeg_encode: needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    res = {"gpu": q, "n": a.n}
    bgr = smooth_frames(a.n, 1080, 1920, 0)
    dev_bgr = [torch.from_numpy(f).cuda() for f in bgr[:4]]
    c = Call([dev_bgr[i % 4] for i in range(a.n)], "bgr")
    res["bgr_1080p_ms"] = time_call(c, a.reps)
    res["bgr_1080p_bytes_per_file"] = float(c.lengths.float().mean())
    del c
    yuv = []
    import cv2
    for f in bgr[:4]:
        i420 = cv2.cvtColor(f, cv2.COLOR_BGR2YUV_I420)
        h, w = 1080, 1920
        uv = np.stack([i420[h:h + h // 4].reshape(h // 2, w // 2), i420[h + h // 4:].reshape(h // 2, w // 2)], 2).reshape(h // 2, w)
        yuv.append(torch.from_numpy(np.concatenate([i420[:h], uv])).cuda())
    c = Call([yuv[i % 4] for i in range(a.n)], "nv12")
    res["nv12_1080p_ms"] = time_call(c, a.reps)
    del c
    raw = []
    for f in bgr[:4]:                                  # RGGB: R at (even, even), B at (odd, odd), G elsewhere
        m = f[..., 1].copy()
        m[0::2, 0::2], m[1::2, 1::2] = f[0::2, 0::2, 2], f[1::2, 1::2, 0]
        raw.append(torch.from_numpy(m).cuda())
    for layout in ("bayer_bg", "bayer_bg_ea"):
        c = Call([raw[i % 4] for i in range(a.n)], layout)
        res[layout + "_1080p_ms"] = time_call(c, a.reps)
        res[layout + "_1080p_bytes_per_file"] = float(c.lengths.float().mean())
        del c
    rng = np.random.RandomState(1)
    regions = []
    for k in range(a.n):
        w, h = int(rng.randint(16, 400)), int(rng.randint(16, 600))
        regions.append((k % 4, int(rng.randint(0, 1920 - w)), int(rng.randint(0, 1080 - h)), w, h))
    c = Call(dev_bgr, "bgr", regions)
    res["crops_ms"] = time_call(c, a.reps)
    del c
    res["cv2_8threads_bgr_1080p_ms"] = host_cv2(bgr)
    res["cv2_8threads_crops_ms"] = host_cv2([bgr[r[0]][r[2]:r[2] + r[4], r[1]:r[1] + r[3]].copy() for r in regions])
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

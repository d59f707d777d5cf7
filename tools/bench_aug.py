#!/usr/bin/env python
"""Training-batch augmentation on the device: img_aug (utils/datasets.py:63-68) with motion_blur, random_resize and augment_hsv
enabled.

  python tools/bench_aug.py [--batch 256 --size 352 --iters 50 --host-images 16] [--geom]

Times, on a uint8 [batch, 3, size, size] batch resident in HBM, each launch after an L2 flush (a 256 MB memset), with CUDA events
around the launch alone:
  contrast_us           yfv2_aug_contrast_brightness (the existing kernel, out of place);
  hsv_us / resize_us / all_us   yfv2_aug_batch with contrast + augment_hsv, contrast + random_resize, and all three;
  blur_us / blur_all_us  yfv2_aug_batch_blur with motion_blur alone and with all four steps, every image blurred (half of them
                         degree 2, half 3; the reference blurs half of its images, see datasets.py:19);
  *_GBps                 the batch read once plus the batch written once, over the time (the elementwise modes' minimum traffic;
                         the resize modes read about (rw*rh)/(W*H) of each source image more than once, which this does not count).
--geom adds yfv2_aug_geometric (YOLOv5's load_mosaic -> random_perspective with border 114 -> fliplr) to the same run:
  geom_mosaic_affine_us / geom_mosaic_persp_us   every image a mosaic of four batch images, warped by cv2.warpAffine /
                         cv2.warpPerspective matrices drawn with degrees 10, shear 5, scale 0.5, translate 0.1 (perspective
                         5e-4), half of them flipped;
  geom_flip_us           fliplr alone (identity M);
  geom_draws_us / geom_labels_us / geom_host_us   the host side of one batch of 64 mosaics with 8 boxes per image, as the
                         trainer runs it in its main process: utils.device_aug.draw_geometric, geometric_targets, and the two
                         together, medians of 20 (host times, not device times).
host_*_us: the reference's own contrast_and_brightness, motion_blur (blurred images only), random_resize and augment_hsv per
image on one core
(cv2.setNumThreads(1)), when the reference checkout is on PYTHONPATH; otherwise they are reported as not measured.
Prints one JSON line with the GPU name and power limit."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)
import yfv2  # noqa: E402,F401
import torch  # noqa: E402

import yfv2_engine as eng  # noqa: E402


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:                                           # noqa: BLE001
        return "unknown (%s)" % e


def time_launch(fn, iters, flush):
    ts = []
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(iters):
        flush.zero_()
        s.record()
        fn()
        e.record()
        e.synchronize()
        ts.append(s.elapsed_time(e) * 1e3)
    return float(np.median(ts)), float(np.min(ts)), float(np.max(ts))


def host_times(n_img, size):
    try:
        import cv2
        import utils.datasets as ds                                  # the reference's, when its checkout is on PYTHONPATH
        if not hasattr(ds, "augment_hsv"):
            return None
    except Exception:                                                # noqa: BLE001
        return None
    cv2.setNumThreads(1)
    rs = np.random.RandomState(0)
    imgs = [rs.randint(0, 256, (size, size, 3)).astype(np.uint8) for _ in range(n_img)]
    out = {}
    import random

    def blurred(img):                                                # motion_blur with its randint(1, 2) forced to 1
        real = random.randint
        random.randint = lambda lo, hi: 1 if (lo, hi) == (1, 2) else real(lo, hi)
        try:
            return ds.motion_blur(img)
        finally:
            random.randint = real
    for name, fn in (("contrast", ds.contrast_and_brightness), ("motion_blur", blurred), ("random_resize", ds.random_resize),
                     ("augment_hsv", ds.augment_hsv)):
        fn(imgs[0])
        t0 = time.perf_counter()
        for im in imgs:
            fn(im)
        out["host_%s_us" % name] = (time.perf_counter() - t0) / n_img * 1e6
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--size", type=int, default=352)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--host-images", type=int, default=16)
    ap.add_argument("--geom", action="store_true", help="also time yfv2_aug_geometric and the host label step")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_aug.py: needs a CUDA device")
    N, S = args.batch, args.size
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randint(0, 256, (N, 3, S, S), dtype=torch.uint8, device="cuda", generator=g)
    out = torch.empty_like(x)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    rs = np.random.RandomState(1)
    a, b = rs.uniform(0.25, 1.75, N), rs.uniform(0.25, 1.75, N)
    rw = (S * rs.uniform(0.8, 1, N)).astype(int)
    rh = (S * rs.uniform(0.8, 1, N)).astype(int)
    luts = eng.hsv_luts(rs.uniform(-1, 1, (N, 3)) * [0.0138, 0.678, 0.36] + 1)
    at, bt = torch.tensor(a, dtype=torch.float32, device="cuda"), torch.tensor(b, dtype=torch.float32, device="cuda")
    lut_t = torch.from_numpy(luts).cuda()
    params = (eng.AugParams * N)(*[eng.AugParams(float(a[i]), float(b[i]), int(rw[i]), int(rh[i])) for i in range(N)])
    blur = [(2 + i % 2, float(rs.uniform(-360, 360))) for i in range(N)]
    desc = (eng.AugBlur * N)()
    for i, (d, ang) in enumerate(blur):
        desc[i].ksize = d
        for j, v in enumerate(eng.motion_blur_taps(d, ang).ravel()):
            desc[i].taps[j] = float(v)
    nb = ctypes.c_size_t()
    eng._check(eng.lib().yfv2_aug_blur_workspace_bytes(N, S, S, ctypes.byref(nb)), "aug_blur_workspace_bytes")
    ws = torch.empty(nb.value, dtype=torch.uint8, device="cuda")
    L, stream = eng.lib(), eng._stream(x.device)

    def launch(flags):                                               # arguments built once: the events time the launch alone
        p = lambda t: ctypes.c_void_p(t.data_ptr())                  # noqa: E731
        if flags & eng.AUG_BLUR:
            return lambda: eng._check(L.yfv2_aug_batch_blur(p(x), p(out), N, S, S, params, p(lut_t), desc, flags, p(ws), nb.value,
                                                            stream), "aug_batch_blur")
        return lambda: eng._check(L.yfv2_aug_batch(p(x), p(out), N, S, S, params, p(lut_t), flags, stream), "aug_batch")

    modes = {
        "contrast": lambda: eng._check(L.yfv2_aug_contrast_brightness(ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(out.data_ptr()),
                                                                      ctypes.c_void_p(at.data_ptr()), ctypes.c_void_p(bt.data_ptr()),
                                                                      N, 3 * S * S, stream), "contrast"),
        "hsv": launch(eng.AUG_CONTRAST | eng.AUG_HSV),
        "resize": launch(eng.AUG_CONTRAST | eng.AUG_RESIZE),
        "all": launch(eng.AUG_CONTRAST | eng.AUG_RESIZE | eng.AUG_HSV),
        "blur": launch(eng.AUG_BLUR),
        "blur_all": launch(eng.AUG_CONTRAST | eng.AUG_RESIZE | eng.AUG_HSV | eng.AUG_BLUR),
    }
    assert torch.equal(eng.augment_batch(x, a, b, rw, rh, luts), (modes["all"](), out)[1])      # the timed call is the API's
    assert torch.equal(eng.augment_batch(x, blur=blur), (modes["blur"](), out)[1])
    assert torch.equal(eng.augment_batch(x, a, b, rw, rh, luts, blur=blur), (modes["blur_all"](), out)[1])
    if args.geom:
        import random
        import utils.device_aug as da
        draws = {
            "geom_mosaic_affine": da.draw_geometric(N, S, S, random.Random(2), mosaic=1.0, degrees=10, shear=5),
            "geom_mosaic_persp": da.draw_geometric(N, S, S, random.Random(3), mosaic=1.0, degrees=10, shear=5, perspective=0.0005),
            "geom_flip": [dict(M=np.eye(3), perspective=False, mosaic=False, src=[i] * 4, flip=True) for i in range(N)],
        }
        for name, d in draws.items():
            modes[name] = (lambda gd: lambda: eng._check(L.yfv2_aug_geometric(ctypes.c_void_p(x.data_ptr()),
                                                                               ctypes.c_void_p(out.data_ptr()), N, S, S, gd,
                                                                               stream), "aug_geometric"))(eng.geom_descriptors(d))
            assert torch.equal(eng.augment_geometric(x, d), (modes[name](), out)[1])
        assert torch.equal(out, torch.flip(x, [3]))
    res = {"gpu": gpu_info(), "batch": N, "size": S, "iters": args.iters}
    moved = 2 * x.numel()
    for name, fn in modes.items():
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        med, lo, hi = time_launch(fn, args.iters, flush)
        res[name + "_us"] = round(med, 1)
        res[name + "_us_range"] = [round(lo, 1), round(hi, 1)]
        res[name + "_GBps"] = round(moved / med / 1e3, 1)
    res["bytes_moved"] = moved
    if args.geom:
        import random
        import utils.device_aug as da
        rs = np.random.RandomState(4)
        t = np.concatenate([np.column_stack([np.full(8, n), rs.randint(0, 80, 8), rs.uniform(0.1, 0.9, (8, 2)),
                                             rs.uniform(0.05, 0.4, (8, 2))]) for n in range(64)]).astype(np.float32)
        tt = torch.from_numpy(t)
        ts = []
        for i in range(21):
            t0 = time.perf_counter()
            d = da.draw_geometric(64, S, S, random.Random(5 + i), mosaic=1.0, degrees=10, shear=5)
            t1 = time.perf_counter()
            da.geometric_targets(tt, d, S, S)
            ts.append((t1 - t0, time.perf_counter() - t1))
        ts = np.array(ts[1:]) * 1e6
        res["geom_draws_us"] = round(float(np.median(ts[:, 0])), 1)
        res["geom_labels_us"] = round(float(np.median(ts[:, 1])), 1)
        res["geom_host_us"] = round(float(np.median(ts.sum(1))), 1)
    ht = host_times(args.host_images, S)
    res.update({k: round(v, 1) for k, v in ht.items()} if ht else {"host": "reference checkout not on PYTHONPATH: not measured"})
    print(json.dumps(res))


if __name__ == "__main__":
    main()

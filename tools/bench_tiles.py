#!/usr/bin/env python
"""Tiled detection on full-HD frames: 3 x 2 tiles at overlap 0.2 plus the whole frame (7 network images per frame), per-region
resize + forward + fused decode/NMS, then one yfv2_merge_regions call that maps the rows to frame pixels and removes duplicates
across regions.

  python tools/bench_tiles.py [--steps K --warmup W --frames 256 --cols 3 --rows 2 --overlap 0.2 --runs 2]

256 seeded 1920x1080 BGR frames resident in HBM, two batches alternated; bench.py's random weights (they keep 300 rows per region
image, so 2100 candidates per frame: the merge's worst case at the reference's cap) and thresholds.  The region images run in
chunks of 256 (the plan bench.py uses).  Prints one JSON line with, per run:
  frames_per_s     frames over the device time of whole steps (CUDA events);
  step_ms          one step: resize + forward + decode/NMS of every region image, and the merge;
  resize_ms, forward_ms, decode_nms_ms: each phase of a step on its own (CUDA events, all chunks);
  merge_us         the merge launch alone, L2 flushed before each launch, and merge_share_of_step.
The card's name and power limit are read in the same process; frames 0 and F-1 of the last warm-up step are checked against
tests/region_oracle.py bit for bit."""
import argparse
import ctypes
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)
import bench  # noqa: E402
import torch  # noqa: E402


def events_ms(fn, n, stream):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(n):
        fn()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--cols", type=int, default=3)
    ap.add_argument("--rows", type=int, default=2)
    ap.add_argument("--overlap", type=float, default=0.2)
    ap.add_argument("--merge", default="ios", choices=("ios", "iou"))
    ap.add_argument("--merge-thres", type=float, default=0.5)
    ap.add_argument("--max-det", type=int, default=1000)
    ap.add_argument("--runs", type=int, default=2)
    args = ap.parse_args()
    import yfv2  # noqa: F401
    import yfv2_engine as eng
    import region_oracle as ro
    from utils.frames import tile_regions
    if not torch.cuda.is_available():
        raise SystemExit("bench_tiles.py: no CUDA device (the product path has no CPU fallback)")
    F, S, CH = args.frames, bench.SIDE, bench.BATCH
    fw, fh = 1920, 1080
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    model, _ = bench.random_state_dict()
    model = model.to(dev).eval()
    c = bench.cfg()
    L = eng.lib()
    stream = torch.cuda.current_stream(dev)
    sp = ctypes.c_void_p(stream.cuda_stream)

    g = torch.Generator(device=dev).manual_seed(3)
    frames = [torch.randint(0, 256, (F, fh, fw, 3), generator=g, dtype=torch.uint8, device=dev) for _ in range(2)]
    tiles = tile_regions(fw, fh, args.cols, args.rows, args.overlap, True)
    regions = [(f,) + t for f in range(F) for t in tiles]
    T = len(regions)
    descs = []                      # the crops as yfv2_frame descriptors (views: pixel (x0, y0) of the frame, the frame's pitch)
    for fb in frames:
        d = (eng.Frame * T)()
        for k, (f, x0, y0, w, h) in enumerate(regions):
            pitch = fb[f].stride(0)
            d[k].data, d[k].w, d[k].h, d[k].pitch = fb[f].data_ptr() + y0 * pitch + 3 * x0, w, h, pitch
        descs.append(d)
    rdesc = (eng.Region * T)(*[eng.Region(*r) for r in regions])
    x = torch.empty((T, 3, S, S), dtype=torch.uint8, device=dev)
    plan = model._plan_for(x[:CH])
    preds = [plan.alloc_preds() for _ in range(0, T, CH)]
    anchors = eng.anchors_array(c)
    M = eng.MAX_DET
    dets = torch.empty((T, M, 6), dtype=torch.float32, device=dev)
    counts = torch.empty((T,), dtype=torch.int32, device=dev)
    out = torch.empty((F, args.max_det, 6), dtype=torch.float64, device=dev)
    out_counts = torch.empty((F,), dtype=torch.int32, device=dev)
    kept = torch.empty((F, args.max_det), dtype=torch.int32, device=dev)
    metric = eng.MERGE_METRICS[args.merge]
    it = [0]
    chunks = [(k, min(CH, T - k)) for k in range(0, T, CH)]
    if any(n != CH for _, n in chunks):
        raise SystemExit("bench_tiles.py: %d region images are not a whole number of %d-image chunks" % (T, CH))

    def ok(rc_):
        if rc_:
            raise RuntimeError(L.yfv2_last_error())

    def resize():
        ok(L.yfv2_resize_bgr_u8(descs[it[0] % 2], T, S, S, ctypes.c_void_p(x.data_ptr()), sp))

    def forward():
        for (k, n), p in zip(chunks, preds):
            plan.forward(x[k:k + n], p)

    def decode_nms():
        for (k, n), p in zip(chunks, preds):
            ok(L.yfv2_decode_nms(eng._ptr_array(p), n, S, S, bench.ANCHORS, bench.CLASSES, anchors, ctypes.c_float(bench.CONF),
                                 ctypes.c_double(bench.IOU), None, 0, M, ctypes.c_float(eng.MAX_WH),
                                 ctypes.c_void_p(dets[k].data_ptr()), ctypes.c_void_p(counts[k:].data_ptr()), None, None, sp))

    def merge():
        ok(L.yfv2_merge_regions(ctypes.c_void_p(dets.data_ptr()), ctypes.c_void_p(counts.data_ptr()), rdesc, T, M, F, S, S,
                                ctypes.c_double(args.merge_thres), metric, args.max_det, ctypes.c_void_p(out.data_ptr()),
                                ctypes.c_void_p(out_counts.data_ptr()), ctypes.c_void_p(kept.data_ptr()), sp))

    def step():
        resize()
        forward()
        decode_nms()
        merge()
        it[0] += 1

    for _ in range(max(args.warmup, 2)):
        step()
    torch.cuda.synchronize(dev)
    # parity of the timed path's merge: frames 0 and F-1 of the last step against the oracle, bit for bit
    d_h, n_h = dets.cpu().numpy(), counts.cpu().numpy()
    o_h, c_h, k_h = out.cpu().numpy(), out_counts.cpu().numpy(), kept.cpu().numpy()
    per = len(tiles)
    for f in (0, F - 1):
        sl = slice(f * per, (f + 1) * per)
        wo, wc, wk = ro.merge(d_h[sl], n_h[sl], [(0,) + r[1:] for r in regions[sl]], 1, S, S, args.merge_thres, metric, args.max_det)
        if not (wc[0] == c_h[f] and np.array_equal(o_h[f].view(np.uint64), wo[0].view(np.uint64))
                and np.array_equal(np.where(wk[0] >= 0, wk[0] + f * per * M, -1), k_h[f])):
            raise AssertionError("bench_tiles parity: frame %d differs from tests/region_oracle.py" % f)
    candidates = int(n_h.sum())

    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)     # 256 MB > L2
    sampler = bench.ClockSampler(0)
    sampler.start()
    runs = []
    for _ in range(args.runs):
        ms_step = events_ms(step, args.steps, stream)
        phase = {}
        for name, fn in (("resize_ms", resize), ("forward_ms", forward), ("decode_nms_ms", decode_nms)):
            phase[name] = round(events_ms(fn, args.steps, stream) / args.steps, 4)
        tot, reps = 0.0, max(5, min(args.steps, 20))
        for _ in range(reps):
            flush.zero_()
            tot += events_ms(merge, 1, stream)
        us = 1e3 * tot / reps
        runs.append(dict({"step_ms": round(ms_step / args.steps, 4), "frames_per_s": round(F * args.steps / (ms_step * 1e-3), 1),
                          "network_images_per_s": round(T * args.steps / (ms_step * 1e-3), 1), "merge_us": round(us, 2),
                          "merge_share_of_step": round(us * 1e-3 / (ms_step / args.steps), 4)}, **phase))
    clocks = sampler.stop()
    power = None
    try:
        import pynvml
        pynvml.nvmlInit()
        power = pynvml.nvmlDeviceGetPowerManagementLimit(pynvml.nvmlDeviceGetHandleByIndex(0)) / 1000.0
    except Exception:
        pass
    line = {"metric": "frames/sec %dx%d frames, %dx%d tiles + full frame -> per-region detect at %dx%d + merge"
                      % (fw, fh, args.cols, args.rows, S, S),
            "value": runs[-1]["frames_per_s"], "unit": "frames/s", "steps": args.steps, "frames": F, "regions_per_frame": per,
            "network_images_per_step": T, "runs": runs, "device": torch.cuda.get_device_name(dev), "power_limit_w": power,
            "clocks": clocks, "candidates_per_frame": candidates / F, "kept_per_frame": float(c_h.mean()),
            "merge": args.merge, "merge_thres": args.merge_thres, "max_det": args.max_det,
            "timing": "CUDA events; frames resident in HBM, two batches alternated; merge_us with L2 flushed before each launch",
            "parity": "merged rows, counts and kept_src of frames 0 and %d equal tests/region_oracle.py bit for bit" % (F - 1)}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()

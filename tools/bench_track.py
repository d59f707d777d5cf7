#!/usr/bin/env python
"""The multi-stream tracker on the device (yfv2_track_update), alone and inside track_frames.

  python tools/bench_track.py [--steps K --warmup W --runs 5 --frames 256]

1. The update alone, 256 streams and 16 streams of seeded scenes (60 objects per stream moving linearly with noise; each frame 50
   of them high-score and 10 low-score, plus 10 low-score clutter rows, so 50 high and 20 low detections and about 60 live
   tracks per stream; capacity 128).  The frames are generated once and
   resident in HBM; a run times `steps` consecutive updates with CUDA events; the two sizes alternate run by run and each reports
   the median of its runs.
2. track_frames on `frames` full-HD NV12 frames of a pan over tests/golden/000139.jpg (decoded and stretched to 1920x1080 on the
   device, shifted 4 px per frame, converted to NV12 with BT.601 studio-range integer arithmetic) with the model-zoo weights:
   one step split into resize, forward, decode/NMS and track (scale to frame pixels + update), each phase timed with CUDA events
   over `steps` repetitions.
The card's name and power limit are read in the same process.  Prints one JSON line."""
import argparse
import json
import os
import statistics
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


def scenes(S, T, seed, n_obj=60, n_high=50, n_clutter=10):
    """[T, S, n_obj + n_clutter, 6] float64 rows: n_obj objects per stream in linear motion, n_high of them high-score each frame
    and the others low-score, then n_clutter low-score rows at random places."""
    rng = np.random.default_rng(seed)
    p = rng.uniform([100, 100], [1800, 980], (S, n_obj, 2))
    v = rng.normal(0, 4, (S, n_obj, 2))
    wh = rng.uniform([20, 40], [80, 160], (S, n_obj, 2))
    out = np.zeros((T, S, n_obj, 6))
    for t in range(T):
        c = p + v * t + rng.normal(0, 1.5, p.shape)
        hi = np.argsort(rng.random((S, n_obj)), axis=1) < n_high
        out[t, :, :, 0:2] = c - wh / 2
        out[t, :, :, 2:4] = c + wh / 2
        out[t, :, :, 4] = np.where(hi, rng.uniform(0.6, 0.95, (S, n_obj)), rng.uniform(0.15, 0.45, (S, n_obj)))
        out[t, :, :, 5] = 0.0
    cl = rng.uniform([0, 0, 10, 10], [1900, 1060, 40, 40], (T, S, n_clutter, 4))
    junk = np.concatenate([cl[..., :2], cl[..., :2] + cl[..., 2:], rng.uniform(0.15, 0.45, (T, S, n_clutter, 1)),
                           np.zeros((T, S, n_clutter, 1))], axis=-1)
    return np.concatenate([out, junk], axis=2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--frames", type=int, default=256)
    args = ap.parse_args()
    import yfv2  # noqa: F401
    import yfv2_engine as eng
    from utils.tracking import track_frames
    if not torch.cuda.is_available():
        raise SystemExit("bench_track.py: no CUDA device (the product path has no CPU fallback)")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    stream = torch.cuda.current_stream(dev)

    # 1. the update alone
    T = args.warmup + args.steps * args.runs
    setups = {}
    for S in (256, 16):
        dets = torch.from_numpy(scenes(S, T, seed=S)).to(dev)
        counts = torch.full((S,), dets.shape[2], dtype=torch.int32, device=dev)
        tr = eng.Tracker(dev, S, 128)
        for t in range(args.warmup):
            tr.update(dets[t], counts)
        setups[S] = dict(dets=dets, counts=counts, tr=tr, t=args.warmup, ms=[], live=[])
    for _ in range(args.runs):
        for S, st in setups.items():
            def one(st=st):
                st["last"] = st["tr"].update(st["dets"][st["t"]], st["counts"])
                st["t"] += 1
            st["ms"].append(events_ms(one, args.steps, stream) / args.steps)
            st["live"].append(float(st["last"][1].double().mean()))
    update = {str(S): {"update_us_median": round(1e3 * statistics.median(st["ms"]), 2),
                       "update_us_runs": [round(1e3 * m, 2) for m in st["ms"]],
                       "streams_per_s": round(S / (statistics.median(st["ms"]) * 1e-3), 1),
                       "confirmed_tracks_per_stream": round(statistics.mean(st["live"]), 1)} for S, st in setups.items()}

    # 2. track_frames on full-HD NV12 frames, phase by phase
    import model.detector as det
    import synth
    from utils.frames import read_images
    golden = os.path.join(ROOT, "tests", "golden")
    model = det.Detector(80, 3, True)
    model.load_state_dict({k: torch.from_numpy(v) for k, v in synth.load_modelzoo_weights(golden).items()})
    model = model.to(dev).eval()
    c = synth.coco_cfg()
    F, fw, fh = args.frames, 1920, 1080
    img = read_images([os.path.join(golden, "000139.jpg")])[0]
    bgr = eng.resize_frames([img], fw, fh, "bgr", dev)[0].int()                       # [3, fh, fw]
    buf = torch.empty((F, fh * 3 // 2, fw), dtype=torch.uint8, device=dev)
    for i in range(F):
        b, g_, r = torch.roll(bgr, 4 * i, dims=2)
        buf[i, :fh] = ((66 * r + 129 * g_ + 25 * b + 128) >> 8) + 16
        sub = lambda p: p.reshape(fh // 2, 2, fw // 2, 2).float().mean((1, 3)).round().int()     # noqa: E731
        rs, gs, bs = sub(r), sub(g_), sub(b)
        uv = buf[i, fh:].view(fh // 2, fw // 2, 2)
        uv[..., 0] = (((-38 * rs - 74 * gs + 112 * bs + 128) >> 8) + 128).clamp(0, 255)
        uv[..., 1] = (((112 * rs - 94 * gs - 18 * bs + 128) >> 8) + 128).clamp(0, 255)
    frames = [buf[i] for i in range(F)]
    tracker = eng.Tracker(dev, F, 128)
    for _ in range(max(args.warmup, 2)):
        track_frames(model, tracker, frames, c, layout="nv12")
    torch.cuda.synchronize(dev)
    x = eng.resize_frames(frames, c["width"], c["height"], "nv12", dev)
    with torch.no_grad():
        preds = model(x)
    rows, counts, _ = eng.decode_nms(preds, c, tracker.low_thresh, 0.4)
    scale = torch.tensor([fw / c["width"], fh / c["height"]] * 2 + [1.0, 1.0], dtype=torch.float64, device=dev)

    def resize():
        eng.resize_frames(frames, c["width"], c["height"], "nv12", dev, out=x)

    def forward():
        with torch.no_grad():
            model(x)

    def decode():
        eng.decode_nms(preds, c, tracker.low_thresh, 0.4)

    def track():
        tracker.update(rows.double() * scale, counts)

    def whole():
        track_frames(model, tracker, frames, c, layout="nv12")

    phases = {}
    for name, fn in (("step_ms", whole), ("resize_ms", resize), ("forward_ms", forward), ("decode_nms_ms", decode), ("track_ms", track)):
        phases[name] = round(events_ms(fn, args.steps, stream) / args.steps, 4)
    phases["track_share_of_step"] = round(phases["track_ms"] / phases["step_ms"], 4)
    phases["rows_per_frame"] = float(counts.double().mean())
    power = None
    try:
        import pynvml
        pynvml.nvmlInit()
        power = pynvml.nvmlDeviceGetPowerManagementLimit(pynvml.nvmlDeviceGetHandleByIndex(0)) / 1000.0
    except Exception:
        pass
    line = {"metric": "yfv2_track_update us per call (capacity 128, 50 high + 20 low rows per stream)", "update": update,
            "track_frames": dict(phases, frames=F, size="%dx%d nv12" % (fw, fh)), "steps": args.steps, "runs": args.runs,
            "device": torch.cuda.get_device_name(dev), "power_limit_w": power,
            "timing": "CUDA events; update sizes alternated run by run, medians; track_frames phases each over `steps` repetitions"}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()

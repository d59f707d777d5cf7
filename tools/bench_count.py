#!/usr/bin/env python
"""The line and zone counter on the device (yfv2_count_update), with the tracker update it follows for scale.

  python tools/bench_count.py [--steps K --warmup W --runs 5]

1. 16, 256 and 4096 streams of seeded scenes (60 objects per stream in linear motion with noise, 50 high-score and 10 low-score
   each frame, plus 10 low-score clutter rows, so about 60 confirmed tracks per stream; capacity 128), each stream with its own
   seeded geometry: 4 lines and 4 zones of 8 vertices.  The detections are generated on the device.  Each frame runs
   yfv2_track_update, then yfv2_count_update (E = 64); each call is timed with its own pair of CUDA events, and a run sums
   `steps` frames.  The sizes alternate run by run and each reports the median of its runs.
2. tests/count_oracle.py, the contract restated on the host, on the 16-stream scene driven by tests/track_oracle.py: host
   seconds per frame of the count step alone.
The card's name and power limit are read in the same process.  Prints one JSON line."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)
import bench  # noqa: E402,F401
import torch  # noqa: E402


def geometry(rng):
    lines = [tuple(rng.uniform([0, 0, 0, 0], [1920, 1080, 1920, 1080]).tolist()) for _ in range(4)]
    zones = []
    for _ in range(4):
        a = np.sort(rng.uniform(0, 2 * np.pi, 8))
        c, r = rng.uniform([200, 200], [1700, 880]), rng.uniform(60, 300, 8)
        zones.append(np.stack([c[0] + r * np.cos(a), c[1] + r * np.sin(a)], 1).astype(np.float32))
    return lines, zones


class Scene:
    """S streams of n_obj objects in linear motion on the device; frame(t) fills the [S, n_obj + n_clutter, 6] rows."""

    def __init__(self, S, seed, dev, n_obj=60, n_high=50, n_clutter=10):
        self.g = torch.Generator(device=dev).manual_seed(seed)
        u = lambda *shape: torch.rand(shape, generator=self.g, device=dev, dtype=torch.float64)     # noqa: E731
        self.u, self.S, self.n_obj, self.n_high, self.n_clutter = u, S, n_obj, n_high, n_clutter
        self.p = torch.stack([100 + 1700 * u(S, n_obj), 100 + 880 * u(S, n_obj)], -1)
        self.v = (u(S, n_obj, 2) - 0.5) * 8
        self.wh = torch.stack([20 + 60 * u(S, n_obj), 40 + 120 * u(S, n_obj)], -1)
        self.rows = torch.zeros((S, n_obj + n_clutter, 6), dtype=torch.float64, device=dev)
        self.counts = torch.full((S,), n_obj + n_clutter, dtype=torch.int32, device=dev)

    def frame(self, t):
        S, n, u = self.S, self.n_obj, self.u
        c = self.p + self.v * t + (u(S, n, 2) - 0.5) * 3
        hi = torch.argsort(u(S, n), 1) < self.n_high
        self.rows[:, :n, 0:2] = c - self.wh / 2
        self.rows[:, :n, 2:4] = c + self.wh / 2
        self.rows[:, :n, 4] = torch.where(hi, 0.6 + 0.35 * u(S, n), 0.15 + 0.3 * u(S, n))
        cl = u(S, self.n_clutter, 4) * torch.tensor([1900, 1060, 30, 30], dtype=torch.float64, device=self.rows.device)
        self.rows[:, n:, 0:2] = cl[..., :2]
        self.rows[:, n:, 2:4] = cl[..., :2] + 10 + cl[..., 2:]
        self.rows[:, n:, 4] = 0.15 + 0.3 * u(S, self.n_clutter)
        return self.rows, self.counts


def timed(fn, stream):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    r = fn()
    e1.record(stream)
    return e0, e1, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--oracle-frames", type=int, default=5)
    args = ap.parse_args()
    import yfv2  # noqa: F401
    import yfv2_engine as eng
    if not torch.cuda.is_available():
        raise SystemExit("bench_count.py: no CUDA device (the product path has no CPU fallback)")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    stream = torch.cuda.current_stream(dev)

    # 1. the count update, and the tracker update it follows
    setups = {}
    for S in (16, 256, 4096):
        rng = np.random.default_rng(S)
        tr = eng.Tracker(dev, S, 128)
        ct = eng.Counter(tr, max_lines=4, max_zones=4, max_vertices=8)
        for s in range(S):
            ct.set_geometry(s, *geometry(rng))
        sc = Scene(S, S, dev)
        for t in range(args.warmup):
            tr.update(*sc.frame(t))
            ct.update(max_events=64)
        setups[S] = dict(tr=tr, ct=ct, sc=sc, t=args.warmup, count=[], track=[], tracks=[], events=[])
    for _ in range(args.runs):
        for S, st in setups.items():
            marks = []
            for _ in range(args.steps):
                rows, counts = st["sc"].frame(st["t"])
                st["t"] += 1
                a = timed(lambda: st["tr"].update(rows, counts), stream)
                b = timed(lambda: st["ct"].update(max_events=64), stream)
                marks.append((a, b))
            torch.cuda.synchronize(dev)
            st["track"].append(sum(a[0].elapsed_time(a[1]) for a, _ in marks) / args.steps)
            st["count"].append(sum(b[0].elapsed_time(b[1]) for _, b in marks) / args.steps)
            st["tracks"].append(float(marks[-1][0][2][1].double().mean()))
            st["events"].append(float(marks[-1][1][2][1].double().mean()))
    update = {str(S): {"count_us_median": round(1e3 * statistics.median(st["count"]), 2),
                       "count_us_runs": [round(1e3 * m, 2) for m in st["count"]],
                       "track_us_median": round(1e3 * statistics.median(st["track"]), 2),
                       "confirmed_tracks_per_stream": round(statistics.mean(st["tracks"]), 1),
                       "events_per_stream_per_frame": round(statistics.mean(st["events"]), 3)} for S, st in setups.items()}

    # 2. the oracle's host time per frame, 16 streams
    import count_oracle as co
    import track_cases as tc
    import track_oracle as to
    case = tc.scene(1, S=16, frames=args.oracle_frames + 3, K=128, max_objects=60)
    want_t, want = to.Tracker(16, 128, **case["params"]), co.Counter(16)
    rng = np.random.default_rng(16)
    for s in range(16):
        want.set_geometry(s, *geometry(rng))
    host = []
    for step in case["steps"]:
        d, n = tc.to_arrays(step[2])
        want_t.update(d, n, step[1])
        t0 = time.perf_counter()
        want.update(want_t, step[1])
        host.append((time.perf_counter() - t0) / len(step[1]) * 16)
    power = None
    try:
        import pynvml
        pynvml.nvmlInit()
        power = pynvml.nvmlDeviceGetPowerManagementLimit(pynvml.nvmlDeviceGetHandleByIndex(0)) / 1000.0
    except Exception:
        pass
    line = {"metric": "yfv2_count_update us per call (4 lines, 4 zones of 8 vertices per stream; capacity 128)", "update": update,
            "oracle_host_ms_per_frame_16_streams": round(1e3 * statistics.median(host[3:] or host), 2),
            "steps": args.steps, "runs": args.runs, "device": torch.cuda.get_device_name(dev), "power_limit_w": power,
            "timing": "CUDA events around each call; sizes alternated run by run, medians"}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()

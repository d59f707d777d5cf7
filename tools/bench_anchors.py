"""Anchor k-means on the device at COCO train2017 scale: 860 k seeded lognormal boxes, k = 6, R restarts in one batch.

    python tools/bench_anchors.py [--boxes 860000 --k 6 --restarts 1,16,64]

Per R, one JSON line: end-to-end seconds of yfv2_engine.kmeans_anchors (host clock around the call, which ends in a device
synchronise), the iterations of the longest run (each run's are listed), ms per iteration, and the kernels' device time per
iteration from torch.profiler in a separate 10-iteration run (assign, update = ordered sums + centroid update, avg IoU once).
Then the numpy oracle's host time per iteration (oracle/anchors.py: assign + ordered sums) and the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import yfv2  # noqa: E402,F401
import yfv2_engine  # noqa: E402
import anchor_cases as ac  # noqa: E402
from oracle import anchors as oa  # noqa: E402
from utils import anchors as ua  # noqa: E402


def kernel_ms(X, k, init, iters):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        yfv2_engine.kmeans_anchors(X, k, init, iters)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for name in ("anchor_assign_kernel", "anchor_update_kernel", "anchor_avg_iou_kernel"):
            if name in e.key:
                out[name] = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--boxes", type=int, default=860_000)
    ap.add_argument("--k", type=int, default=6)
    ap.add_argument("--restarts", default="1,16,64")
    ap.add_argument("--oracle-iters", type=int, default=3)
    args = ap.parse_args()
    X = ac.lognormal(args.boxes, 2017)
    k = args.k
    yfv2_engine.kmeans_anchors(X[:10000], k, np.arange(k)[None], 3)       # load the module, warm the allocator
    torch.cuda.synchronize()
    for R in [int(r) for r in args.restarts.split(",")]:
        init = ua.initial_picks(ua.seeded_rng(R), X.shape[0], k, R)
        yfv2_engine.kmeans_anchors(X, k, init, 2)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = yfv2_engine.kmeans_anchors(X, k, init)
        torch.cuda.synchronize()
        e2e = time.perf_counter() - t0
        iters = res.iterations.cpu().numpy()
        km = kernel_ms(X, k, init, 10)
        print(json.dumps({"R": R, "N": X.shape[0], "k": k, "e2e_s": round(e2e, 4), "iterations_max": int(iters.max()),
                          "iterations": iters.tolist(), "status": res.status.cpu().numpy().tolist(),
                          "ms_per_iteration": round(1e3 * e2e / int(iters.max()), 3),
                          "assign_ms_per_iteration": round(km.get("anchor_assign_kernel", 0.0) / 10, 3),
                          "update_ms_per_iteration": round(km.get("anchor_update_kernel", 0.0) / 10, 3),
                          "avg_iou_ms": round(km.get("anchor_avg_iou_kernel", 0.0), 3)}), flush=True)
    C = X[ua.initial_picks(ua.seeded_rng(0), X.shape[0], k)[0]]
    t0 = time.perf_counter()
    for _ in range(args.oracle_iters):
        a = oa.assign(X, C)
        C, _ = oa.update(X, a, k)
    host = (time.perf_counter() - t0) / args.oracle_iters
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"oracle_numpy_s_per_iteration": round(host, 3), "gpu": torch.cuda.get_device_name(),
                      "nvidia_smi": smi.stdout.strip()}), flush=True)


if __name__ == "__main__":
    main()

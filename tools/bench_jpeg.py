#!/usr/bin/env python
"""JPEG decode on the device (yfv2_engine.decode_jpeg) at batch: 256 and 1024 files of the reference's two photos (500x334 and
500x375, 4:2:0, no restart markers) repeated, and of the 1920x1080 4:2:0 fixture (tests/golden/jpeg_cases.npz).

  python tools/bench_jpeg.py [--batches 256,1024 --reps 5] [--progressive]

--progressive runs the same rows on progressive files (decode_jpeg(progressive=True)): the two photos re-coded losslessly as
progressive files with cv2's script (tests/golden/jpeg_progressive.npz, tx_cv2_*: the same coefficients as the baseline rows'
photos) and the progressive 1080p fixture, and adds entropy_level_ms (the entropy phase's kernels per level, from
torch.profiler) and blob_bytes_per_file.

Prints one JSON line per (files, batch) with:
  parse_ms        yfv2_jpeg_parse of the batch on the host (one core; both calls: sizes, then the blob), median;
  decode_ms       decode_jpeg end to end: pack into pinned memory, parse, one H2D copy, the three launches, the error-flag read back
                  (host clock around work that ends in a synchronise), median;
  entropy_ms, idct_ms, color_ms: each phase alone on the parsed, resident batch, CUDA events, median;
  img_per_s       files / decode_ms;
  detect_ms       (photos, first batch only) utils.frames.detect_files end to end from paths, 352x352, the reference's thresholds;
  nvjpeg_ms       torchvision.io.decode_jpeg(device="cuda") of the same files when torchvision is importable; NOT bit-exact with
                  cv2 (nvJPEG's IDCT and upsampling), listed for scale only.
The GPU's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)
import torch  # noqa: E402
import yfv2  # noqa: E402,F401
import yfv2_engine as eng  # noqa: E402


def gpu():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name()


def host_ms(fn, reps):
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t) * 1e3)
    return float(np.median(ts))


def event_ms(fn, reps):
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def level_ms(fn, reps):
    """Median device time of each prog_entropy_kernel launch of fn (one per level, in launch order), from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    runs = []
    for _ in range(reps):
        with profile(activities=[ProfilerActivity.CUDA]) as p:
            fn()
            torch.cuda.synchronize()
        ev = sorted((e for e in p.events() if "prog_entropy_kernel" in e.name and e.device_type.name == "CUDA"),
                    key=lambda e: e.time_range.start)
        runs.append([e.time_range.elapsed_us() / 1e3 for e in ev])
    n = max(len(r) for r in runs)                            # the profiler can drop an event of a rep: medians of complete reps
    full = [r for r in runs if len(r) == n]
    return [float(np.median([r[k] for r in full])) for k in range(n)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="256,1024")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--progressive", action="store_true")
    args = ap.parse_args()
    gdir = os.path.join(ROOT, "tests", "golden")
    prog = args.progressive
    if prog:
        pg = np.load(os.path.join(gdir, "jpeg_progressive.npz"))
        photos = [pg["jpg_tx_cv2_" + s] for s in ("000139", "000004")]
        fullhd = [pg["jpg_cv2_fullhd_420"]]
    else:
        photos = [np.fromfile(os.path.join(gdir, s + ".jpg"), np.uint8) for s in ("000139", "000004")]
        fullhd = [np.load(os.path.join(gdir, "jpeg_cases.npz"))["jpg_fullhd_420"]]
    try:
        import torchvision.io as tvio
    except Exception:                                      # noqa: BLE001  (nvJPEG is optional context)
        tvio = None
    card = gpu()
    tmp = tempfile.mkdtemp(prefix="bench_jpeg_")
    for label, src in (("photos", photos), ("fullhd", fullhd)):
        for bi, n in enumerate(int(b) for b in args.batches.split(",")):
            files = [src[i % len(src)] for i in range(n)]
            kw = {"progressive": True} if prog else {}
            eng.decode_jpeg(files[:8], "cuda", **kw)                        # warm-up: module load
            res = {"files": label + ("_progressive" if prog else ""), "batch": n, "bytes_per_file": int(np.mean([f.size for f in files])),
                   "gpu": card}
            res["parse_ms"] = host_ms(lambda: eng.parse_jpeg(files, blob=True, **kw), args.reps)
            res["decode_ms"] = host_ms(lambda: eng.decode_jpeg(files, "cuda", **kw), args.reps)
            b = eng.JpegBatch(files, "cuda", **kw)
            b.decode()
            b.check()
            for ph, key in ((eng.JPEG_ENTROPY, "entropy_ms"), (eng.JPEG_IDCT, "idct_ms"), (eng.JPEG_COLOR, "color_ms")):
                res[key] = event_ms(lambda: b.decode(ph), args.reps)
            res["segments"] = sum(i["segments"] for i in b.infos)
            if prog:
                res["scans"] = sum(i["scans"] for i in b.infos)
                res["blob_bytes_per_file"] = b.blob.numel() // n
                res["entropy_level_ms"] = level_ms(lambda: b.decode(eng.JPEG_ENTROPY), args.reps)
            del b
            res["img_per_s"] = n / res["decode_ms"] * 1e3
            if label == "photos" and bi == 0:
                import model.detector as det
                import synth
                import utils.frames as uf
                paths = []
                for i, f in enumerate(files):
                    paths.append(os.path.join(tmp, "%d.jpg" % i))
                    f.tofile(paths[-1])
                torch.manual_seed(1)
                m = det.Detector(80, 3, True).cuda().eval()
                cfg = synth.coco_cfg()
                uf.detect_files(m, paths[:8], cfg, **kw)
                res["detect_ms"] = host_ms(lambda: uf.detect_files(m, paths, cfg, 0.3, 0.4, **kw), args.reps)
            if tvio is not None:
                ts = [torch.from_numpy(f) for f in files]
                tvio.decode_jpeg(ts[:8], device="cuda")
                res["nvjpeg_ms"] = host_ms(lambda: tvio.decode_jpeg(ts, device="cuda"), args.reps)
                res["nvjpeg_note"] = "torchvision nvJPEG, not bit-exact with cv2.imread"
            torch.cuda.empty_cache()
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()

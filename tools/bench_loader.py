#!/usr/bin/env python
"""Training and evaluation input from image files: the fused JPEG decode + resize and the device loader (DESIGN.md §13).

  python tools/bench_loader.py [--files 2048 --batch 256 --reps 10 --train-batch 64]

Prints one JSON line per measurement, and the GPU's name and power limit read in the same run:
  (a) kernel   batch 256 at 352x352, CUDA events, median of calls alternated one by one: the fused call (decode_resize: entropy,
               IDCT, fused colour + resize) against decode + resize_bgr (entropy, IDCT, colour into the arena, resize), on the
               reference's two photos repeated and on the 1080p fixture; entropy + IDCT, colour and resize alone; fused_phase_ms is
               the fused call minus entropy + IDCT (derived, not timed alone);
  (b) loader   images/s from files on local disk (the two photos copied --files times, seeded labels) through DataLoader
               (8 workers, collate_files) + DeviceLoader to a synchronised CUDA batch, second epoch (workers warm);
  (c) host     the same files through cv2.imread + cv2.resize in 8 workers (TensorDataset(imgaug=False)'s work), when cv2 is
               importable; otherwise "not measured";
  (d) train    train_dist.py --device-decode --device-aug steps/s on those files (the time of a 30-iteration run minus that of a
               10-iteration one, over 20, after a 5-iteration warm-up run; all inside the first epoch: 2048 files / batch 64 = 32
               iterations), and the same run fed by the reference's TensorDataset when utils.datasets (the reference checkout) and
               cv2 are importable; otherwise "not measured"."""
import argparse
import json
import os
import shutil
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

GOLDEN = os.path.join(ROOT, "tests", "golden")


def gpu():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name()


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def kernels(name, files, reps, W=352, H=352):
    bt = eng.JpegBatch(files, "cuda")
    bt.decode()
    fr = bt.frames()
    out = torch.empty((len(files), 3, H, W), dtype=torch.uint8, device="cuda")
    res = torch.empty_like(out)
    two = lambda: (bt.decode(), eng.resize_bgr(fr, W, H, out=res))      # noqa: E731
    fused = lambda: bt.decode_resize(out, W, H)                         # noqa: E731
    for _ in range(3):
        two(), fused()
    assert torch.equal(out, res) and not any(bt.flags())
    t = {"two_call_ms": [], "fused_ms": [], "entropy_idct_ms": [], "color_ms": [], "resize_ms": []}
    for _ in range(reps):                                               # alternated call by call
        t["two_call_ms"].append(timed(two))
        t["fused_ms"].append(timed(fused))
        t["entropy_idct_ms"].append(timed(lambda: bt.decode(eng.JPEG_ENTROPY | eng.JPEG_IDCT)))
        t["color_ms"].append(timed(lambda: bt.decode(eng.JPEG_COLOR)))
        t["resize_ms"].append(timed(lambda: eng.resize_bgr(fr, W, H, out=res)))
    m = {k: round(float(np.median(v)), 3) for k, v in t.items()}
    m["fused_phase_ms"] = round(m["fused_ms"] - m["entropy_idct_ms"], 3)
    m["color_plus_resize_ms"] = round(m["color_ms"] + m["resize_ms"], 3)
    return dict(measurement="a_kernel", workload=name, batch=len(files), size="%dx%d" % (W, H), reps=reps, **m)


def make_dataset(root, n):
    rng = np.random.default_rng(5)
    names = []
    for i in range(n):
        src = os.path.join(GOLDEN, ("000004", "000139")[i % 2] + ".jpg")
        name = os.path.join(root, "img%05d.jpg" % i)
        shutil.copyfile(src, name)
        with open(os.path.join(root, "img%05d.txt" % i), "w") as f:
            for _ in range(int(rng.integers(1, 8))):
                f.write("%d %.6f %.6f %.6f %.6f\n" % (int(rng.integers(0, 80)), *rng.uniform(0.1, 0.9, 4)))
        names.append(name)
    lst = os.path.join(root, "list.txt")
    with open(lst, "w") as f:
        f.write("".join(n + "\n" for n in names))
    return lst


def epoch_rate(it_factory, n):
    """Images/s of the second pass over a loader (workers started and warm), ending in a synchronise."""
    rates = []
    for _ in range(2):
        torch.cuda.synchronize()
        t = time.perf_counter()
        seen = 0
        for imgs, _ in it_factory():
            seen += imgs.shape[0]
        torch.cuda.synchronize()
        rates.append(seen / (time.perf_counter() - t))
    assert seen == n
    return round(rates[-1], 1)


class HostDataset(torch.utils.data.Dataset):
    """TensorDataset(imgaug=False)'s image work: cv2.imread + cv2.resize(INTER_LINEAR) + transpose (datasets.py:106-110)."""

    def __init__(self, lst, W, H):
        with open(lst) as f:
            self.paths = [ln.strip() for ln in f if ln.strip()]
        self.W, self.H = W, H

    def __len__(self):
        return len(self.paths)

    def __getitem__(self, i):
        import cv2
        img = cv2.resize(cv2.imread(self.paths[i]), (self.W, self.H), interpolation=cv2.INTER_LINEAR)
        return torch.from_numpy(img.transpose(2, 0, 1).copy()), torch.zeros((0,))


def train_rate(data, extra):
    import train_dist
    ts = []
    for iters in (5, 10, 30):                   # the first run warms up what the process does once (modules, graphs)
        torch.cuda.synchronize()
        t = time.perf_counter()
        train_dist.main(["--data", data, "--device-aug", "--max-iters", str(iters)] + extra)
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t)
    return round(20 / (ts[2] - ts[1]), 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=2048)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--train-batch", type=int, default=64)
    a = ap.parse_args()
    print(json.dumps({"gpu": gpu()}), flush=True)

    photos = []
    for p in ("000004", "000139"):
        with open(os.path.join(GOLDEN, p + ".jpg"), "rb") as f:
            photos.append(f.read())
    print(json.dumps(kernels("photos_500x334_500x375_420", [photos[i % 2] for i in range(a.batch)], a.reps)), flush=True)
    hd = np.load(os.path.join(GOLDEN, "jpeg_cases.npz"))["jpg_fullhd_420"].tobytes()
    print(json.dumps(kernels("fixture_1920x1080_420", [hd] * a.batch, a.reps)), flush=True)

    from utils.device_data import device_loader
    root = tempfile.mkdtemp(prefix="yfv2_bench_loader_")
    try:
        lst = make_dataset(root, a.files)
        dl = device_loader(lst, 352, 352, a.batch, torch.device("cuda"), num_workers=8)
        print(json.dumps({"measurement": "b_device_loader", "files": a.files, "batch": a.batch, "workers": 8,
                          "img_per_s": epoch_rate(lambda: dl, a.files)}), flush=True)
        try:
            import cv2  # noqa: F401
            host = torch.utils.data.DataLoader(HostDataset(lst, 352, 352), batch_size=a.batch, num_workers=8, pin_memory=True,
                                               persistent_workers=True)
            rate = epoch_rate(lambda: ((x.cuda(non_blocking=True), t) for x, t in host), a.files)
        except ImportError:
            rate = "not measured"
        print(json.dumps({"measurement": "c_host_cv2_loader", "files": a.files, "batch": a.batch, "workers": 8, "img_per_s": rate}),
              flush=True)

        weights = os.path.join(root, "w.pth")
        import synth
        torch.save({k: torch.from_numpy(v) for k, v in synth.load_modelzoo_weights(GOLDEN).items()}, weights)
        data = os.path.join(root, "bench.data")
        with open(data, "w") as f:
            f.write("[name]\nmodel_name=coco\n\n[train-configure]\nepochs=3\nsteps=150,250\nbatch_size=%d\nsubdivisions=1\n"
                    "learning_rate=0.001\n\n[model-configure]\npre_weights=%s\nclasses=80\nwidth=352\nheight=352\nanchor_num=3\n"
                    "anchors=12.64,19.39, 37.88,51.48, 55.71,138.31, 126.91,78.23, 131.57,214.55, 279.92,258.87\n\n"
                    "[data-configure]\ntrain=%s\nval=%s\nnames=none\n" % (a.train_batch, weights, lst, lst))
        dev = train_rate(data, ["--device-decode", "--save-dir", root])
        try:
            import cv2  # noqa: F401
            import utils.datasets  # noqa: F401
            host = train_rate(data, ["--save-dir", root])
        except ImportError:
            host = "not measured (no reference utils.datasets or cv2 here)"
        print(json.dumps({"measurement": "d_train_dist", "batch": a.train_batch, "device_decode_steps_per_s": dev,
                          "host_loader_steps_per_s": host}), flush=True)
    finally:
        shutil.rmtree(root, ignore_errors=True)
    print(json.dumps({"gpu": gpu()}), flush=True)


if __name__ == "__main__":
    main()

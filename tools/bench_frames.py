#!/usr/bin/env python
"""Raw-frame inference: device resize (yfv2_resize_bgr_u8) + forward + fused decode/NMS from 1920x1080 BGR frames resident in HBM.

  python tools/bench_frames.py [--steps K --warmup W --batch 256 --frame 1920x1080 --runs 2 --layout bgr|nv12|i420|rgb|...]

Same network, weights (Detector default init under seed 1), target size and NMS thresholds as bench.py.  Two frame batches
(2 x 1.6 GB at batch 256) are alternated so that no step reads its frames from the 50 MB L2.  Prints one JSON line with, per run:
  step_ms         resize + forward + decode/NMS per batch, CUDA events over K steps;
  step_ms_noresize the same steps from an already resized uint8 batch (bench.py's timed step), so the resize's share is visible;
  resize_us       the resize launch alone, L2 flushed before each launch, CUDA events;
  resize_GBps / resize_frac: the bytes the resize touches over resize_us, against the HBM peak.
Touched bytes are counted from the coefficients: 32-byte sectors of every source row the kernel reads (the two rows and the two
columns of each output pixel) plus the planar output written.  `h2d_ms_per_batch` is one pinned host->device copy of a frame
batch: frames that start on the host are bound by that copy (about 6.2 MB per frame), not by the kernel.

--layout nv12 | i420 feeds the steps YUV 4:2:0 frames of the same size (cv2's single [h*3/2, w] buffer) through
yfv2_resize_yuv420_u8 instead; --layout rgb | bgra | rgba | gray | rgb_chw feeds contiguous frames of that layout through
yfv2_resize_strided_u8, and --layout yuyv | uyvy | yvyu packed 4:2:2 frames through yfv2_resize_yuv422_u8.  Each run then also
times the BGR resize of the same frame size (bgr_resize_us), alternated launch by launch with the layout's resize, each after an
L2 flush; the touched bytes count the sectors of the rows (and planes) the layout's resize reads; `h2d_ms_per_batch` is the pinned
copy of a batch in that layout next to `h2d_bgr_ms_per_batch`; and the parity check runs tests/layout_oracle.py on frames 0 and
N-1."""
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


def touched_bytes(h, w, H, W, pitch):
    """Bytes of DRAM sectors one frame's resize reads (each 32-byte sector once) plus the bytes it writes."""
    from oracle import resize as ore
    sx, _, _ = ore.coeffs(w, W, True)
    sy, _, _ = ore.coeffs(h, H, False)
    cols = np.unique(np.concatenate([sx, np.minimum(sx + 1, w - 1)]))
    rows = np.unique(np.clip(np.concatenate([sy, sy + 1]), 0, h - 1))
    byte = (3 * cols[:, None] + np.arange(3)[None, :]).reshape(-1)
    sectors = len(np.unique((rows[:, None] * pitch + byte[None, :]) // 32))
    return 32 * sectors + 3 * H * W


def touched_bytes_yuv420(h, w, H, W, layout):
    """The same count for one YUV 4:2:0 single-buffer frame (rows w bytes apart): the sectors of the luma rows and chroma rows the
    kernel reads (two rows, two columns and their chroma per output pixel) plus the bytes it writes."""
    from oracle import resize as ore
    sx, _, _ = ore.coeffs(w, W, True)
    sy, _, _ = ore.coeffs(h, H, False)
    cols = np.unique(np.concatenate([sx, np.minimum(sx + 1, w - 1)]))
    rows = np.unique(np.clip(np.concatenate([sy, sy + 1]), 0, h - 1))
    crows, ccols = np.unique(rows >> 1), np.unique(cols >> 1)
    addr = [(rows[:, None] * w + cols[None, :]).reshape(-1)]
    if layout == "nv12":
        addr.append((h * w + crows[:, None] * w + (2 * ccols[:, None] + np.arange(2)[None, :]).reshape(-1)[None, :]).reshape(-1))
    else:
        for plane in (h * w, h * w + (h // 2) * (w // 2)):
            addr.append((plane + crows[:, None] * (w // 2) + ccols[None, :]).reshape(-1))
    return 32 * len(np.unique(np.concatenate(addr) // 32)) + 3 * H * W


def touched_bytes_layout(h, w, H, W, layout):
    """The same count for one contiguous frame of a strided or packed 4:2:2 layout: the sectors of the bytes the kernel reads for
    the two rows and two columns of each output pixel (three channel bytes; for 4:2:2 the luma and the macropixel's U and V),
    plus the bytes it writes."""
    from oracle import resize as ore
    import layout_oracle as lo
    sx, _, _ = ore.coeffs(w, W, True)
    sy, _, _ = ore.coeffs(h, H, False)
    cols = np.unique(np.concatenate([sx, np.minimum(sx + 1, w - 1)]))[None, :]
    rows = np.unique(np.clip(np.concatenate([sy, sy + 1]), 0, h - 1))[:, None]
    if layout == "rgb_chw":
        addr = [p * h * w + rows * w + cols for p in range(3)]
    elif layout in lo.MACROPIXEL:
        oy, ou, _, ov = lo.MACROPIXEL[layout]
        addr = [rows * 2 * w + 2 * cols + oy, rows * 2 * w + 4 * (cols >> 1) + ou, rows * 2 * w + 4 * (cols >> 1) + ov]
    else:
        step = {"rgb": 3, "bgra": 4, "rgba": 4, "gray": 1}[layout]
        addr = [rows * step * w + step * cols + o for o in ((0,) if layout == "gray" else (0, 1, 2))]
    return 32 * len(np.unique(np.concatenate([a.reshape(-1) for a in addr]) // 32)) + 3 * H * W


def layout_descs(fb, layout):
    """Descriptors of a [N, ...] batch of contiguous frames of a strided or packed 4:2:2 layout, and the entry that takes them."""
    import yfv2_engine as eng
    N = fb.shape[0]
    if layout in eng.YUV422_LAYOUTS:
        d = (eng.Yuv422Frame * N)()
        oy, ou, ov = eng._YUV422_OFFSETS[layout]
        for i in range(N):
            p = fb[i].data_ptr()
            d[i].y, d[i].u, d[i].v, d[i].pitch, d[i].h, d[i].w = p + oy, p + ou, p + ov, fb[i].stride(0), fb.shape[1], fb.shape[2]
        return d, eng.lib().yfv2_resize_yuv422_u8
    d = (eng.StridedFrame * N)()
    for i in range(N):
        p = fb[i].data_ptr()
        if layout == "rgb_chw":
            s = fb[i].stride(0)
            d[i].b, d[i].g, d[i].r, d[i].pitch, d[i].step = p + 2 * s, p + s, p, fb[i].stride(1), 1
            d[i].h, d[i].w = fb.shape[2], fb.shape[3]
        else:
            ob, og, or_ = eng._BGR_OFFSETS[layout]
            step = 1 if layout == "gray" else fb.shape[3]
            d[i].b, d[i].g, d[i].r, d[i].pitch, d[i].step = p + ob, p + og, p + or_, fb[i].stride(0), step
            d[i].h, d[i].w = fb.shape[1], fb.shape[2]
    return d, eng.lib().yfv2_resize_strided_u8


def yuv420_descs(fb, layout):
    """Descriptors of a [N, h*3/2, w] batch of single-buffer NV12 or I420 frames."""
    import yfv2_engine as eng
    N, rows, w = fb.shape
    h = rows // 3 * 2
    d = (eng.Yuv420Frame * N)()
    for i in range(N):
        base = fb[i].data_ptr()
        d[i].y, d[i].y_pitch, d[i].w, d[i].h = base, w, w, h
        if layout == "nv12":
            d[i].u, d[i].v, d[i].uv_pitch, d[i].uv_step = base + h * w, base + h * w + 1, w, 2
        else:
            d[i].u, d[i].v, d[i].uv_pitch, d[i].uv_step = base + h * w, base + h * w + (h // 2) * (w // 2), w // 2, 1
    return d


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
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--frame", default="1920x1080", help="source frame WxH")
    ap.add_argument("--runs", type=int, default=2, help="measurement runs, alternated within one process")
    ap.add_argument("--layout", default="bgr", choices=("bgr", "nv12", "i420", "rgb", "bgra", "rgba", "gray", "rgb_chw", "yuyv",
                                                        "uyvy", "yvyu"), help="source frame format")
    args = ap.parse_args()
    import yfv2  # noqa: F401
    import yfv2_engine as eng
    from oracle import resize as ore
    if not torch.cuda.is_available():
        raise SystemExit("bench_frames.py: no CUDA device (the product path has no CPU fallback)")
    fw, fh = (int(v) for v in args.frame.lower().split("x"))
    N, S = args.batch, bench.SIDE
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    model, _ = bench.random_state_dict()
    model = model.to(dev).eval()
    c = bench.cfg()
    L = eng.lib()
    stream = torch.cuda.current_stream(dev)
    sp = ctypes.c_void_p(stream.cuda_stream)

    g = torch.Generator(device=dev).manual_seed(3)
    frames = [torch.randint(0, 256, (N, fh, fw, 3), generator=g, dtype=torch.uint8, device=dev) for _ in range(2)]
    descs = []
    for fb in frames:
        d = (eng.Frame * N)()
        for i in range(N):
            d[i].data, d[i].w, d[i].h, d[i].pitch = fb[i].data_ptr(), fw, fh, fb[i].stride(0)
        descs.append(d)
    other = args.layout != "bgr"
    yuv420 = args.layout in ("nv12", "i420")
    if other:
        import layout_cases as lc
        import layout_oracle as lo
        shape = (fh * 3 // 2, fw) if yuv420 else lc.frame_shape(args.layout, fh, fw)
        yframes = [torch.randint(0, 256, (N,) + shape, generator=g, dtype=torch.uint8, device=dev) for _ in range(2)]
        if yuv420:
            ydescs = [yuv420_descs(fb, args.layout) for fb in yframes]
            yentry = L.yfv2_resize_yuv420_u8
        else:
            ydescs = [layout_descs(fb, args.layout)[0] for fb in yframes]
            yentry = layout_descs(yframes[0][:1], args.layout)[1]
    x = torch.empty((N, 3, S, S), dtype=torch.uint8, device=dev)
    plan = model._plan_for(x)
    preds = plan.alloc_preds()
    anchors = eng.anchors_array(c)
    out = torch.empty((N, eng.MAX_DET, 6), dtype=torch.float32, device=dev)
    counts = torch.empty((N,), dtype=torch.int32, device=dev)
    it = [0]

    def resize_bgr():
        rc = L.yfv2_resize_bgr_u8(descs[it[0] % 2], N, S, S, ctypes.c_void_p(x.data_ptr()), sp)
        if rc:
            raise RuntimeError(L.yfv2_last_error())

    def resize_other():
        rc = yentry(ydescs[it[0] % 2], N, S, S, ctypes.c_void_p(x.data_ptr()), sp)
        if rc:
            raise RuntimeError(L.yfv2_last_error())

    resize = resize_other if other else resize_bgr

    def detect():
        plan.forward(x, preds)
        rc = L.yfv2_decode_nms(eng._ptr_array(preds), N, S, S, bench.ANCHORS, bench.CLASSES, anchors, ctypes.c_float(bench.CONF),
                               ctypes.c_double(bench.IOU), None, 0, eng.MAX_DET, ctypes.c_float(eng.MAX_WH),
                               ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(counts.data_ptr()), None, None, sp)
        if rc:
            raise RuntimeError(L.yfv2_last_error())

    def step():
        resize()
        detect()
        it[0] += 1

    for _ in range(max(args.warmup, 3)):
        step()
    torch.cuda.synchronize(dev)
    # parity of the timed path's resize: first and last frame of the batch the last warm-up step resized, against the oracle
    last = (yframes if other else frames)[(it[0] - 1) % 2]
    for i in (0, N - 1):
        src = last[i].cpu().numpy()
        want = lo.resize_planar(src, args.layout, S, S) if other else ore.resize_bgr_planar(src, S, S)
        if not np.array_equal(x[i].cpu().numpy(), want):
            raise AssertionError("bench_frames parity: resized frame %d differs from the oracle" % i)

    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)     # 256 MB > L2
    per_frame = touched_bytes(fh, fw, S, S, frames[0][0].stride(0))
    if other:
        per_frame_bgr, per_frame = per_frame, (touched_bytes_yuv420(fh, fw, S, S, args.layout) if yuv420 else
                                               touched_bytes_layout(fh, fw, S, S, args.layout))
    peak, peak_src = bench.measured_peak()
    sampler = bench.ClockSampler(0)
    sampler.start()
    runs = []
    for _ in range(args.runs):
        ms_step = events_ms(step, args.steps, stream)
        ms_det = events_ms(detect, args.steps, stream)
        tot, tot_bgr, reps = 0.0, 0.0, max(5, min(args.steps, 20))
        for _ in range(reps):
            flush.zero_()
            it[0] += 1
            tot += events_ms(resize, 1, stream)
            if other:                      # the BGR resize of the same frame size, alternated launch by launch
                flush.zero_()
                tot_bgr += events_ms(resize_bgr, 1, stream)
        us = 1e3 * tot / reps
        gbs = N * per_frame / (us * 1e-6) / 1e9
        runs.append({"step_ms": round(ms_step / args.steps, 4), "step_ms_noresize": round(ms_det / args.steps, 4),
                     "images_per_s": round(N * args.steps / (ms_step * 1e-3), 1), "resize_us": round(us, 2),
                     "resize_share_of_step": round(us * 1e-3 / (ms_step / args.steps), 4),
                     "resize_GBps": round(gbs, 1), "resize_frac": round(gbs / peak, 4)})
        if other:
            us_bgr = 1e3 * tot_bgr / reps
            runs[-1].update({"bgr_resize_us": round(us_bgr, 2),
                             "bgr_resize_GBps": round(N * per_frame_bgr / (us_bgr * 1e-6) / 1e9, 1)})
    clocks = sampler.stop()
    del flush

    host = torch.empty((N, fh, fw, 3), dtype=torch.uint8, pin_memory=True)
    h2d = [events_ms(lambda: frames[0].copy_(host, non_blocking=True), 1, stream) for _ in range(3)]
    if other:
        del host
        yhost = torch.empty((N,) + shape, dtype=torch.uint8, pin_memory=True)
        h2d_bgr, h2d = h2d, [events_ms(lambda: yframes[0].copy_(yhost, non_blocking=True), 1, stream) for _ in range(3)]
    power = None
    try:
        import pynvml
        pynvml.nvmlInit()
        power = pynvml.nvmlDeviceGetPowerManagementLimit(pynvml.nvmlDeviceGetHandleByIndex(0)) / 1000.0
    except Exception:
        pass
    line = {"metric": "images/sec %dx%d frames -> resize + fwd + decode + NMS at %dx%d" % (fw, fh, S, S),
            "value": runs[-1]["images_per_s"], "unit": "images/s", "steps": args.steps, "batch": N, "runs": runs,
            "device": torch.cuda.get_device_name(dev), "power_limit_w": power, "clocks": clocks,
            "resize_touched_bytes_per_frame": per_frame, "resize_touched_bytes_per_batch": N * per_frame,
            "frame_bytes": fh * fw * 3, "peak_GBps": peak, "peak_source": peak_src,
            "timing": "CUDA events; frames resident in HBM, two batches alternated; resize_us with L2 flushed before each launch",
            "h2d_ms_per_batch": round(min(h2d), 3),
            "h2d_note": "one pinned host->device copy of %d frames (%.1f MB): the bound for frames that start on the host"
                        % (N, N * fh * fw * 3 / 1e6),
            "parity": "resized frames 0 and %d equal the oracle (oracle/resize.py) byte for byte" % (N - 1),
            "kept_boxes_per_step": int(counts.sum().item())}
    if other:
        line["metric"] = "images/sec %dx%d %s frames -> resize + fwd + decode + NMS at %dx%d" % (fw, fh, args.layout.upper(), S, S)
        frame_bytes = int(np.prod(shape))
        line.update({"layout": args.layout, "frame_bytes": frame_bytes, "bgr_frame_bytes": fh * fw * 3,
                     "bgr_resize_touched_bytes_per_frame": per_frame_bgr, "h2d_bgr_ms_per_batch": round(min(h2d_bgr), 3),
                     "timing": line["timing"] + "; bgr_resize_us: the BGR resize of the same frame size, alternated with it",
                     "h2d_note": "one pinned host->device copy of %d %s frames (%.1f MB); h2d_bgr_ms_per_batch: the same frames as BGR "
                                 "(%.1f MB)" % (N, args.layout.upper(), N * frame_bytes / 1e6, N * fh * fw * 3 / 1e6),
                     "parity": "resized frames 0 and %d equal the oracle (tests/layout_oracle.py) byte for byte" % (N - 1)})
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()

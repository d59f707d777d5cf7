"""Detection on raw frames: what test.py:34-68 does around the network, for a batch of frames of any sizes and layouts.

The reference resizes each frame on the host with cv2.resize (test.py:35), runs the network on the resized batch and scales the
boxes back to the frame with scale_w = w / cfg["width"], scale_h = h / cfg["height"] (test.py:57-68).  Here the resize runs on
the device (resize_bgr: yfv2_resize_bgr_u8, bit-identical to cv2's INTER_LINEAR bytes; resize_yuv420: yfv2_resize_yuv420_u8, the
same after cv2.cvtColor(COLOR_YUV2BGR_*); resize_frames: every layout, RGB, BGRA / RGBA, grey, planar RGB and packed YUV 4:2:2
included, the same after the cv2.cvtColor that brings it to BGR), followed by the uint8 forward and the fused decode + NMS; only
the scale-back of at most 300 rows per frame stays on the host, in float64 like test.py's Python floats.

detect_regions / detect_tiled look at each frame through several regions (tiles, zones): every region is cropped in place,
stretched to the network input and detected on like a frame, and yfv2_merge_regions maps the rows of all regions back to frame
pixels and removes the duplicates across regions on the device (include/yfv2.h, DESIGN.md §8)."""
import math

import torch

import yfv2_engine
from yfv2_engine import crop_frame, frame_size, resize_bgr, resize_frames, resize_yuv420  # noqa: F401  (frames -> [N, 3, H, W] uint8 input)
from utils.utils import detect


def to_source_pixels(rows, size, cfg):
    """[n, 6] (x1, y1, x2, y2, conf, cls) in network-input pixels -> float64 [n, 6] with the corners in pixels of a frame of size
    (h, w): x * (w / cfg["width"]), y * (h / cfg["height"]) (test.py:57-68); conf and cls are unchanged."""
    h, w = size
    scale_h, scale_w = h / cfg["height"], w / cfg["width"]
    out = rows.detach().cpu().double().clone()
    out[:, [0, 2]] *= scale_w
    out[:, [1, 3]] *= scale_h
    return out


def int_corners(rows):
    """The integer corners test.py draws, int(x1), int(y1), int(x2), int(y2) (truncation toward zero), of source-pixel rows."""
    return rows[:, :4].trunc().long()


def _yuv420_size(f):
    """(h, w) of the Y plane of a YUV 4:2:0 frame: a (y, ...) tuple of planes or a single [h*3/2, w] buffer."""
    return frame_size(f, "nv12")


def detect_frames(model, frames, cfg, conf_thres=0.3, iou_thres=0.4, layout="bgr"):
    """Raw frames -> detections in each frame's own pixels: a list of float64 CPU [n_i, 6] tensors (x1, y1, x2, y2, conf, cls),
    descending conf.  model: an eval-mode Detector on a CUDA device; cfg: the load_datafile dict (width, height, anchors).
    layout: one of yfv2_engine.LAYOUTS, or a list with one per frame; the frames are what resize_frames takes for it ("bgr": HWC
    uint8 numpy arrays or CUDA tensors of any sizes; "nv12" | "nv21" | "i420" | "yv12": cv2's single [h*3/2, w] buffer or a tuple
    of planes; "rgb", "bgra" / "rgba", "gray", "rgb_chw" [3, h, w], "yuyv" / "uyvy" / "yvyu" [h, w, 2]), converted as
    cv2.cvtColor(COLOR_<LAYOUT>2BGR) does.  The boxes come back in pixels of each frame's h x w (the luma plane for YUV)."""
    frames = list(frames)
    layouts = [layout] * len(frames) if isinstance(layout, str) else list(layout)
    x = resize_frames(frames, cfg["width"], cfg["height"], layouts, next(model.parameters()).device)
    sizes = [frame_size(f, lay) for f, lay in zip(frames, layouts)]
    with torch.no_grad():
        preds = model(x)
    rows = detect(preds, cfg, conf_thres, iou_thres)
    return [to_source_pixels(r, s, cfg) for r, s in zip(rows, sizes)]


def read_images(paths, device=None, progressive=False):
    """cv2.imread(path) of each JPEG file, decoded on the device (yfv2_engine.decode_jpeg): a list of CUDA uint8 [h, w, 3] BGR
    tensors with cv2's bytes, EXIF orientation applied.  Files outside the subset decode_jpeg supports (progressive unless
    progressive=True, PNG, BMP, ...) raise Yfv2Error naming the path; read those with cv2.imread."""
    paths = [str(p) for p in paths]
    files = []
    for p in paths:
        with open(p, "rb") as f:
            files.append(f.read())
    return yfv2_engine.decode_jpeg(files, device, names=paths, progressive=progressive)


def detect_files(model, paths, cfg, conf_thres=0.3, iou_thres=0.4, progressive=False):
    """What test.py:34-68 computes for each image file: read_images, then detect_frames.  A list of float64 CPU [n_i, 6] tensors
    (x1, y1, x2, y2, conf, cls) in each file's pixels, descending conf.  progressive: read progressive JPEG files too.  The files
    are decoded straight into the network input (JpegBatch.decode_resize: the bytes of read_images + resize_bgr, without the
    full-size frames); they are refused, and raise, as read_images refuses them."""
    paths = [str(p) for p in paths]
    files = []
    for p in paths:
        with open(p, "rb") as f:
            files.append(f.read())
    dev = next(model.parameters()).device
    W, H = int(cfg["width"]), int(cfg["height"])
    b = yfv2_engine.JpegBatch(files, dev, names=paths, progressive=progressive)
    x = torch.empty((len(files), 3, H, W), dtype=torch.uint8, device=dev)
    b.decode_resize(x, W, H)
    b.check()
    with torch.no_grad():
        preds = model(x)
    rows = detect(preds, cfg, conf_thres, iou_thres)
    return [to_source_pixels(r, (i["h"], i["w"]), cfg) for r, i in zip(rows, b.infos)]


def _axis_tiles(n, k, overlap, even):
    """Origins and size of k tiles along an axis of n pixels (see tile_regions)."""
    size = min(n, math.ceil(n / (k - (k - 1) * overlap)))
    if even:
        size = min(n, size + (size & 1))
    x0 = [(i * (n - size)) // (k - 1) if k > 1 else 0 for i in range(k)]
    if even:
        x0 = [x & ~1 for x in x0]
    return x0, size


def tile_regions(w, h, cols, rows, overlap=0.2, full_frame=True, layout="bgr"):
    """A cols x rows grid of overlapping tiles of a w x h frame, as a list of (x0, y0, tw, th), row by row.
    tw = ceil(w / (cols - (cols - 1) * overlap)), at most w (th likewise), and tile k starts at floor(k * (w - tw) / (cols - 1)), so
    the last tile ends on the frame's edge and adjacent tiles overlap by at least overlap * tw - 2 pixels.  For the 4:2:0 layouts
    origins are rounded down and sizes up to even numbers on both axes, for packed 4:2:2 along x only (what crop_frame needs).
    full_frame: the whole frame comes first, as one more region for objects larger than a tile (first, it wins ties of conf).
    Each tile is stretched to the network input like a whole frame."""
    cols, rows, w, h = int(cols), int(rows), int(w), int(h)
    if cols < 1 or rows < 1 or w < 1 or h < 1 or not (0.0 <= overlap < 1.0):
        raise ValueError("tile_regions: need cols, rows, w, h >= 1 and 0 <= overlap < 1, got %d x %d tiles of %d x %d, overlap %r"
                         % (cols, rows, w, h, overlap))
    even_x = layout in yfv2_engine.YUV420_LAYOUTS or layout in yfv2_engine.YUV422_LAYOUTS
    even_y = layout in yfv2_engine.YUV420_LAYOUTS
    xs, tw = _axis_tiles(w, cols, overlap, even_x)
    ys, th = _axis_tiles(h, rows, overlap, even_y)
    tiles = [(x0, y0, tw, th) for y0 in ys for x0 in xs]
    return ([(0, 0, w, h)] if full_frame else []) + tiles


def detect_regions(model, frames, cfg, regions, conf_thres=0.3, iou_thres=0.4, layout="bgr", merge="ios", merge_thres=0.5,
                   max_det=1000, batch=256):
    """Detections on regions of frames, merged per frame: a list of float64 CPU [n_i, 6] tensors (x1, y1, x2, y2, conf, cls) in
    pixels of each frame, descending conf, like detect_frames.  regions: one list of (x0, y0, w, h) per frame (may be empty).
    Each region is cropped in place (crop_frame), stretched to cfg's width x height by resize_frames, run through the uint8 forward
    and the fused decode + NMS (conf_thres, iou_thres, 300 rows per region), in chunks of at most `batch` region images.  The rows
    of all regions then go through one yfv2_merge_regions call: mapped to frame pixels, sorted by conf, and a row is dropped when a
    kept row of ANOTHER region and the same class overlaps it by more than merge_thres ("ios": intersection over the smaller box,
    which removes the part of an object cut by a tile's edge; "iou"); at most max_det rows per frame.  Host frames are copied to
    the device once; nothing is copied back before the merge.  With one whole-frame region per frame this is detect_frames."""
    frames = list(frames)
    layouts = [layout] * len(frames) if isinstance(layout, str) else list(layout)
    regions = [list(r) for r in regions]
    if len(layouts) != len(frames) or len(regions) != len(frames):
        raise yfv2_engine.Yfv2Error("detect_regions: %d frames, %d layouts, %d region lists" % (len(frames), len(layouts), len(regions)))
    if merge not in yfv2_engine.MERGE_METRICS:
        raise yfv2_engine.Yfv2Error("detect_regions: merge must be 'iou' or 'ios', got %r" % (merge,))
    if int(batch) < 1:
        raise yfv2_engine.Yfv2Error("detect_regions: batch must be >= 1, got %r" % (batch,))
    dev = next(model.parameters()).device
    W, H = int(cfg["width"]), int(cfg["height"])
    crops, lays, descs = [], [], []
    for i, (f, lay, regs) in enumerate(zip(frames, layouts, regions)):
        if regs:
            f = _on_device(f, lay, dev)
        for (x0, y0, w, h) in regs:
            crops.append(crop_frame(f, lay, x0, y0, w, h))
            lays.append(lay)
            descs.append((i, x0, y0, w, h))
    F, T = len(frames), len(crops)
    if T == 0:
        return [torch.zeros((0, 6), dtype=torch.float64) for _ in range(F)]
    M = yfv2_engine.MAX_DET
    dets = torch.empty((T, M, 6), dtype=torch.float32, device=dev)
    counts = torch.empty((T,), dtype=torch.int32, device=dev)
    batch = int(batch)
    for k in range(0, T, batch):
        x = resize_frames(crops[k:k + batch], W, H, lays[k:k + batch], dev)
        with torch.no_grad():
            preds = model(x)
        out, cnt, _ = yfv2_engine.decode_nms(preds, cfg, conf_thres, iou_thres)
        dets[k:k + batch].copy_(out)
        counts[k:k + batch].copy_(cnt)
    out, n, _ = yfv2_engine.merge_regions(dets, counts, descs, F, W, H, merge_thres, merge, max_det)
    out, n = out.cpu(), n.cpu().tolist()
    return [out[i, :n[i]].clone() for i in range(F)]


def _on_device(f, layout, dev):
    """A frame (or tuple of planes) as CUDA tensors on `dev`: host arrays copied once, CUDA tensors as they are."""
    if isinstance(f, (tuple, list)):
        return tuple(_on_device(p, layout, dev) for p in f)
    if not isinstance(f, torch.Tensor):
        import numpy as np
        f = torch.from_numpy(np.ascontiguousarray(f))
    return f.to(dev)


def detect_tiled(model, frames, cfg, cols, rows, overlap=0.2, full_frame=True, **kw):
    """detect_regions over tile_regions(w, h, cols, rows, overlap, full_frame, layout) of each frame's size."""
    frames = list(frames)
    layout = kw.get("layout", "bgr")
    layouts = [layout] * len(frames) if isinstance(layout, str) else list(layout)
    regions = []
    for f, lay in zip(frames, layouts):
        h, w = frame_size(f, lay)
        regions.append(tile_regions(w, h, cols, rows, overlap, full_frame, lay))
    return detect_regions(model, frames, cfg, regions, **kw)

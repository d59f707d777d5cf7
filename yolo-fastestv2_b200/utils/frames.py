"""Detection on raw frames: what test.py:34-68 does around the network, for a batch of frames of any sizes and layouts.

The reference resizes each frame on the host with cv2.resize (test.py:35), runs the network on the resized batch and scales the
boxes back to the frame with scale_w = w / cfg["width"], scale_h = h / cfg["height"] (test.py:57-68).  Here the resize runs on
the device (resize_bgr: yfv2_resize_bgr_u8, bit-identical to cv2's INTER_LINEAR bytes; resize_yuv420: yfv2_resize_yuv420_u8, the
same after cv2.cvtColor(COLOR_YUV2BGR_*); resize_frames: every layout, RGB, BGRA / RGBA, grey, planar RGB and packed YUV 4:2:2
included, the same after the cv2.cvtColor that brings it to BGR), followed by the uint8 forward and the fused decode + NMS; only
the scale-back of at most 300 rows per frame stays on the host, in float64 like test.py's Python floats."""
import torch

from yfv2_engine import frame_size, resize_bgr, resize_frames, resize_yuv420  # noqa: F401  (frames -> [N, 3, H, W] uint8 input)
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

"""Tracking objects across video frames: detections of each frame linked to the tracks of its stream (camera) on the device.

track_frames runs what detect_frames runs (the device resize, the uint8 forward, the fused decode + NMS), scales the rows to frame
pixels on the device, and gives them to a yfv2_engine.Tracker (yfv2_track_update: ByteTrack's association and lifecycle, one CTA
per stream, include/yfv2.h); one device-to-host copy brings the tracks back.  count_frames then counts line crossings and zone entries, exits and
occupancy with a yfv2_engine.Counter (yfv2_count_update, one CTA per stream) and brings the tracks and counts back in one copy.
To track on tiles of large frames, give detect_regions' merge (yfv2_engine.merge_regions' out / counts) to Tracker.update
directly."""
import torch

import yfv2_engine
from yfv2_engine import frame_size, resize_frames


def _track_device(fn, model, tracker, frames, cfg, streams, layout, conf_thres, iou_thres):
    """detect_frames' device steps, rows scaled to frame pixels, then Tracker.update: (out, counts) on the device."""
    frames = list(frames)
    layouts = [layout] * len(frames) if isinstance(layout, str) else list(layout)
    if len(layouts) != len(frames):
        raise yfv2_engine.Yfv2Error("%s: %d frames, %d layouts" % (fn, len(frames), len(layouts)))
    conf = tracker.low_thresh if conf_thres is None else conf_thres
    dev = next(model.parameters()).device
    x = resize_frames(frames, cfg["width"], cfg["height"], layouts, dev)
    with torch.no_grad():
        preds = model(x)
    rows, counts, _ = yfv2_engine.decode_nms(preds, cfg, conf, iou_thres)
    scale = torch.ones((len(frames), 1, 6), dtype=torch.float64)
    for i, (f, lay) in enumerate(zip(frames, layouts)):
        h, w = frame_size(f, lay)
        scale[i, 0, [0, 2]] = w / cfg["width"]
        scale[i, 0, [1, 3]] = h / cfg["height"]
    dets = rows.double() * scale.to(dev, non_blocking=True)
    out, n, _ = tracker.update(dets, counts, streams)
    return out, n


def track_frames(model, tracker, frames, cfg, streams=None, layout="bgr", conf_thres=None, iou_thres=0.4):
    """One frame for each of the given streams (None: streams 0..len(frames)-1) -> a list of float64 CPU [n_i, 8] tensors, the
    confirmed tracked tracks of each stream in ascending id: (x1, y1, x2, y2, score, cls, track_id, det_row) in the frame's pixels,
    det_row being the row of the frame's detections (descending conf, as detect_frames returns them) the track took.  frames and
    layout are what detect_frames takes; conf_thres defaults to the tracker's low_thresh, so that the low-score detections reach
    the tracker's second stage.  The rows are scaled exactly as to_source_pixels scales them: x * (w / cfg["width"]) and
    y * (h / cfg["height"]), one fp64 product each."""
    out, n = _track_device("track_frames", model, tracker, frames, cfg, streams, layout, conf_thres, iou_thres)
    B, K = out.shape[0], out.shape[1]
    host = torch.cat([n.double().unsqueeze(1), out.reshape(B, -1)], 1).cpu()
    return [host[i, 1:].reshape(K, 8)[:int(host[i, 0])].clone() for i in range(B)]


def count_frames(model, tracker, counter, frames, cfg, streams=None, layout="bgr", conf_thres=None, iou_thres=0.4, max_events=64):
    """track_frames, then counter.update (a yfv2_engine.Counter of `tracker`) on the same streams -> (tracks, events, event_counts,
    occupancy): tracks as track_frames returns them; events a list of float64 CPU [e_i, 8] tensors (kind, index, dir, track_id,
    cls, x, y, frame), e_i = min(event_counts[i], max_events); event_counts int32 [B], every event of the frame; occupancy int32
    [B, counter.Z].  One device-to-host copy brings all of it back."""
    frames = list(frames)
    if counter.tracker is not tracker:
        raise yfv2_engine.Yfv2Error("count_frames: the counter counts another tracker")
    if int(max_events) < 0:
        raise yfv2_engine.Yfv2Error("count_frames: max_events=%d must be >= 0" % int(max_events))
    idx = list(range(len(frames))) if streams is None else [int(s) for s in streams]
    out, n = _track_device("count_frames", model, tracker, frames, cfg, idx, layout, conf_thres, iou_thres)
    events, ecount, occ = counter.update(idx, max_events)
    B, K, E, Z = out.shape[0], out.shape[1], events.shape[1], occ.shape[1]
    host = torch.cat([n.double().unsqueeze(1), ecount.double().unsqueeze(1), occ.double(), out.reshape(B, -1), events.reshape(B, -1)],
                     1).cpu()
    tracks = [host[i, 2 + Z:2 + Z + 8 * K].reshape(K, 8)[:int(host[i, 0])].clone() for i in range(B)]
    evs = [host[i, 2 + Z + 8 * K:].reshape(E, 8)[:min(int(host[i, 1]), E)].clone() for i in range(B)]
    return tracks, evs, host[:, 1].int(), host[:, 2:2 + Z].int()

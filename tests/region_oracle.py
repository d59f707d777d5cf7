"""numpy float64 restatement (test infrastructure) of the cross-region merge of yfv2_merge_regions (include/yfv2.h): the NMS rows
of T region images mapped to frame pixels, sorted, and suppressed greedily across regions, one list per frame.  Every step is the
same IEEE operation as in the kernel: the mapping is a rounded product then a rounded sum, min / max are `a < b ? a : b` /
`a > b ? a : b` with the kept (earlier) row's value first, and the overlap is compared strictly above the threshold, so a NaN
overlap never suppresses."""
import numpy as np


def mn(a, b):
    return np.where(a < b, a, b)


def mx(a, b):
    return np.where(a > b, a, b)


def map_rows(rows, region, W, H):
    """[n, 6] float32 rows in network-input pixels of a region (x0, y0, w, h) -> float64 rows in frame pixels."""
    x0, y0, w, h = region
    sx, sy = np.float64(w) / np.float64(W), np.float64(h) / np.float64(H)
    out = np.asarray(rows, np.float32).astype(np.float64)
    out[:, [0, 2]] = out[:, [0, 2]] * sx + np.float64(x0)
    out[:, [1, 3]] = out[:, [1, 3]] * sy + np.float64(y0)
    return out


def overlap(a, b, metric):
    """Overlap of box a (a kept row) with each row of b [n, 4] (later rows), float64."""
    with np.errstate(all="ignore"):
        iw = mx(0.0, mn(a[2], b[:, 2]) - mx(a[0], b[:, 0]))
        ih = mx(0.0, mn(a[3], b[:, 3]) - mx(a[1], b[:, 1]))
        inter = iw * ih
        aa = (a[2] - a[0]) * (a[3] - a[1])
        ab = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
        den = mn(aa, ab) if metric else (aa + ab) - inter
        return inter / den


def merge(dets, counts, regions, F, W, H, thr, metric, max_det):
    """The whole call.  dets float32 [T, max_det_in, 6], counts int [T], regions T tuples (frame, x0, y0, w, h).  Returns (out
    float64 [F, max_det, 6], counts int32 [F], kept_src int32 [F, max_det]) as yfv2_merge_regions writes them."""
    dets = np.asarray(dets, np.float32)
    T, mdi = dets.shape[0], dets.shape[1]
    metric = {"iou": 0, "ios": 1}.get(metric, metric)
    out = np.zeros((F, max_det, 6), np.float64)
    out_counts = np.zeros(F, np.int32)
    kept_src = np.full((F, max_det), -1, np.int32)
    by_frame = {}
    for t, r in enumerate(regions):
        by_frame.setdefault(int(r[0]), []).append(t)
    for f, ts in by_frame.items():
        boxes, conf, cls, reg, src = [], [], [], [], []
        for t in ts:
            n = min(max(int(counts[t]), 0), mdi)
            rows = dets[t, :n]
            keep = ~np.isnan(rows[:, 4])
            m = map_rows(rows, regions[t][1:], W, H)
            boxes.append(m[keep])
            conf.append(rows[keep, 4])
            cls.append(rows[keep, 5])
            reg.append(np.full(int(keep.sum()), t, np.int64))
            src.append(t * mdi + np.nonzero(keep)[0])
        boxes, conf, cls, reg, src = (np.concatenate(v) for v in (boxes, conf, cls, reg, src))
        # conf descending, ties by region then row (src = t * max_det_in + row grows with both); -0 ties with +0
        order = np.lexsort((src, -conf.astype(np.float64)))
        boxes, conf, cls, reg, src = boxes[order], conf[order], cls[order], reg[order], src[order]
        alive = np.ones(len(conf), bool)
        kept = []
        for i in range(len(conf)):
            if len(kept) == max_det:
                break
            if not alive[i]:
                continue
            kept.append(i)
            later = np.arange(i + 1, len(conf))
            if later.size:
                q = overlap(boxes[i, :4], boxes[later, :4], metric)
                alive[later] &= ~((reg[later] != reg[i]) & (cls[later] == cls[i]) & (q > thr))
        k = np.array(kept, np.int64)
        out[f, :len(k), :4] = boxes[k, :4]
        out[f, :len(k), 4] = conf[k].astype(np.float64)
        out[f, :len(k), 5] = cls[k].astype(np.float64)
        out_counts[f] = len(k)
        kept_src[f, :len(k)] = src[k]
    return out, out_counts, kept_src

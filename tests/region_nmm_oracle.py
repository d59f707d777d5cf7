"""numpy float64 restatement (test infrastructure) of yfv2_merge_regions_nmm (include/yfv2.h): the cross-region merge of
tests/region_oracle.py followed by greedy non-maximum merging.  It uses region_oracle's mapping, overlap and min / max, so every
step is the same IEEE operation as in the kernel: min / max are `a < b ? a : b` / `a > b ? a : b` with the kept row's value (or
the growing box B) first, and the overlap is compared strictly above the threshold, so a NaN overlap neither absorbs nor folds."""
import numpy as np

import region_oracle as ro


def merge_nmm(dets, counts, regions, F, W, H, thr, metric, max_det):
    """yfv2_merge_regions_nmm (include/yfv2.h): region_oracle.merge()'s rows, counts and kept_src, and each kept box grown by greedy non-maximum
    merging.  Every mapped row that is not an output row, rows after the max_det cap included, belongs to the first output row
    before it in the order that matches it by the suppression test (other region, same cls, overlap > thr on the mapped boxes);
    then each output row's box B starts as its own and, over its rows in the order, takes the union with every row whose overlap
    with the current B (B in the kept row's place) is > thr.  Returns (out, counts, kept_src, merged int32 [F, max_det]: the rows
    each box took, 0 past the count)."""
    out, out_counts, kept_src = ro.merge(dets, counts, regions, F, W, H, thr, metric, max_det)
    dets = np.asarray(dets, np.float32)
    mdi = dets.shape[1]
    metric = {"iou": 0, "ios": 1}.get(metric, metric)
    merged = np.zeros((F, max_det), np.int32)
    by_frame = {}
    for t, r in enumerate(regions):
        by_frame.setdefault(int(r[0]), []).append(t)
    for f, ts in by_frame.items():
        n = int(out_counts[f])
        if n == 0:
            continue
        # every mapped row of the frame in merge()'s order (rows of NaN conf dropped)
        boxes, conf, cls, reg, src = [], [], [], [], []
        for t in ts:
            k = min(max(int(counts[t]), 0), mdi)
            rows = dets[t, :k]
            keep = ~np.isnan(rows[:, 4])
            boxes.append(ro.map_rows(rows, regions[t][1:], W, H)[keep])
            conf.append(rows[keep, 4])
            cls.append(rows[keep, 5])
            reg.append(np.full(int(keep.sum()), t, np.int64))
            src.append(t * mdi + np.nonzero(keep)[0])
        boxes, conf, cls, reg, src = (np.concatenate(v) for v in (boxes, conf, cls, reg, src))
        order = np.lexsort((src, -conf.astype(np.float64)))
        boxes, cls, reg, src = boxes[order], cls[order], reg[order], src[order]
        pos = {int(s_): p for p, s_ in enumerate(src)}
        kept = [pos[int(s_)] for s_ in kept_src[f, :n]]              # the output rows' places in the order
        is_kept = np.zeros(len(src), bool)
        is_kept[kept] = True
        # absorb: each non-output row goes to the first output row before it that matches it (blocks of 256 output rows against
        # every row: overlap(a, b) with a [4, 256, 1] gives the [256, rows] pairs, the output row in the kept row's place)
        owner = np.full(len(src), -1, np.int64)
        col = np.arange(len(src))
        for b0 in range(0, n, 256):
            ps = np.array(kept[b0:b0 + 256])
            q = ro.overlap(boxes[ps, :4].T[:, :, None], boxes[:, :4], metric)
            hit = ((reg[None, :] != reg[ps, None]) & (cls[None, :] == cls[ps, None]) & (q > thr) & (col[None, :] > ps[:, None])
                   & ~is_kept[None, :] & (owner < 0)[None, :])
            first = np.argmax(hit, axis=0)
            took = hit.any(axis=0)
            owner[took] = b0 + first[took]
        # fold, all output rows at once: step k takes the k-th row of every group (a group: the rows of one owner, in the order);
        # overlap(B.T, rows) pairs B of each group with its row elementwise, B in the kept row's place
        B = boxes[kept, :4].copy()
        rows = np.nonzero(owner >= 0)[0]
        rows = rows[np.argsort(owner[rows], kind="stable")]
        first = np.searchsorted(owner[rows], owner[rows])            # index in `rows` of each row's group's first row
        rank = np.arange(len(rows)) - first
        for k in range(int(rank.max()) + 1 if len(rows) else 0):
            j = rows[rank == k]
            g = owner[j]
            fold = ro.overlap(B[g].T, boxes[j, :4], metric) > thr
            j, g = j[fold], g[fold]
            B[g] = np.stack([ro.mn(B[g, 0], boxes[j, 0]), ro.mn(B[g, 1], boxes[j, 1]),
                             ro.mx(B[g, 2], boxes[j, 2]), ro.mx(B[g, 3], boxes[j, 3])], 1)
            merged[f, g] += 1
        out[f, :n, :4] = B
    return out, out_counts, kept_src, merged

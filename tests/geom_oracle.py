"""CPU restatement (test infrastructure) of YOLOv5's geometric augmentation as yfv2_aug_geometric runs it: load_mosaic's canvas,
random_perspective's cv2.warpAffine / cv2.warpPerspective with borderValue (114, 114, 114) and np.fliplr, and YOLOv5's own label
lines for the boxes.  The warp reuses tests/warp_oracle.py's inversion and fixed-point coordinates; the sampling is
tests/remap_oracle.py's, except that a tap outside the canvas reads 114 instead of weighing 0.  Pinned to outputs of the real cv2
in tests/golden/geom_cases.npz (tests/golden/make_golden_geom.py)."""
import numpy as np

import remap_oracle as ro
import warp_oracle as wo

BORDER = 114


def canvas(imgs, d):
    """The canvas of one draw (d: mosaic, src, xc, yc) over HWC images [N, H, W, 3]: image src[0], or load_mosaic's 2W x 2H
    layout of src[0..3] around (xc, yc) filled with 114, placed by YOLOv5's x1a .. y2b lines."""
    imgs = np.asarray(imgs)
    if not d["mosaic"]:
        return imgs[d["src"][0]]
    _, h, w, _ = imgs.shape
    xc, yc = d["xc"], d["yc"]
    img4 = np.full((2 * h, 2 * w, 3), BORDER, np.uint8)
    for i, j in enumerate(d["src"]):
        img = imgs[j]
        if i == 0:
            x1a, y1a, x2a, y2a = max(xc - w, 0), max(yc - h, 0), xc, yc
            x1b, y1b, x2b, y2b = w - (x2a - x1a), h - (y2a - y1a), w, h
        elif i == 1:
            x1a, y1a, x2a, y2a = xc, max(yc - h, 0), min(xc + w, 2 * w), yc
            x1b, y1b, x2b, y2b = 0, h - (y2a - y1a), min(w, x2a - x1a), h
        elif i == 2:
            x1a, y1a, x2a, y2a = max(xc - w, 0), yc, xc, min(2 * h, yc + h)
            x1b, y1b, x2b, y2b = w - (x2a - x1a), 0, w, min(y2a - y1a, h)
        else:
            x1a, y1a, x2a, y2a = xc, yc, min(xc + w, 2 * w), min(2 * h, yc + h)
            x1b, y1b, x2b, y2b = 0, 0, min(w, x2a - x1a), min(y2a - y1a, h)
        img4[y1a:y2a, x1a:x2a] = img[y1b:y2b, x1b:x2b]
    return img4


def remap_border(img, map1, map2, border=BORDER):
    """cv2.remap(img, map1, map2, INTER_LINEAR, BORDER_CONSTANT, border) through fixed maps: remap_oracle.remap with every tap
    weighted and a tap outside the image reading `border`."""
    h, w = img.shape[:2]
    x0, y0 = map1[..., 0].astype(np.int64), map1[..., 1].astype(np.int64)
    wt = ro._TABLE[np.asarray(map2).astype(np.int64) & 1023]
    acc = np.zeros(map1.shape[:2] + (3,), np.int64)
    for k, (dy, dx) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
        yy, xx = y0 + dy, x0 + dx
        inside = (yy >= 0) & (yy < h) & (xx >= 0) & (xx < w)
        px = img[np.clip(yy, 0, h - 1), np.clip(xx, 0, w - 1)].astype(np.int64)
        acc += np.where(inside[..., None], px, border) * wt[..., k][..., None]
    return np.clip((acc + (1 << 14)) >> 15, 0, 255).astype(np.uint8)


def warp(img, M, perspective, W, H):
    """cv2.warpAffine(img, M[:2], (W, H), borderValue=114) or cv2.warpPerspective(img, M, (W, H), borderValue=114)."""
    M = np.asarray(M, np.float64)
    persp, m = wo.dst_to_src(M if perspective else M[:2], False)
    return remap_border(img, *wo.warp_maps(m, persp, 0, 0, W, H))


def augment_image(imgs, d):
    """Output image of one draw (d: mosaic, src, xc, yc, M, perspective, flip) over HWC images [N, H, W, 3]: [H, W, 3]."""
    _, H, W, _ = np.asarray(imgs).shape
    out = warp(canvas(imgs, d), d["M"], d["perspective"], W, H)
    return np.ascontiguousarray(np.fliplr(out) if d["flip"] else out)


def augment_planar(batch, draws):
    """yfv2_aug_geometric of a planar [N, 3, H, W] batch: [N, 3, H, W]."""
    hwc = np.ascontiguousarray(np.asarray(batch).transpose(0, 2, 3, 1))
    return np.stack([augment_image(hwc, d).transpose(2, 0, 1) for d in draws])


def box_candidates(box1, box2, wh_thr=2, ar_thr=100, area_thr=0.1, eps=1e-16):
    w1, h1 = box1[2] - box1[0], box1[3] - box1[1]
    w2, h2 = box2[2] - box2[0], box2[3] - box2[1]
    ar = np.maximum(w2 / (h2 + eps), h2 / (w2 + eps))
    return (w2 > wh_thr) & (h2 > wh_thr) & (w2 * h2 / (w1 * h1 + eps) > area_thr) & (ar < ar_thr)


def yolov5_labels(targets, draws, H, W):
    """The targets of the output images as YOLOv5's own lines compute them (load_mosaic's xywhn2xyxy and clip, random_perspective's
    `xy @ M.T` and box_candidates, xyxy2xywhn(clip=True, eps=1e-3), fliplr's 1 - x), with YOLOv5's label rows (class, x, y, w,
    h) float32 and the batch's targets (image, class, cx, cy, w, h) in and out."""
    t = np.asarray(targets, np.float32)
    rows = []
    for n, d in enumerate(draws):
        labels4 = []
        tiles = d["src"] if d["mosaic"] else d["src"][:1]
        for i, j in enumerate(tiles):
            labels = t[t[:, 0] == j][:, 1:].copy()
            padw = (d["xc"] - W if i in (0, 2) else d["xc"]) if d["mosaic"] else 0
            padh = (d["yc"] - H if i in (0, 1) else d["yc"]) if d["mosaic"] else 0
            x = labels[:, 1:]
            y = np.copy(x)
            y[..., 0] = W * (x[..., 0] - x[..., 2] / 2) + padw
            y[..., 1] = H * (x[..., 1] - x[..., 3] / 2) + padh
            y[..., 2] = W * (x[..., 0] + x[..., 2] / 2) + padw
            y[..., 3] = H * (x[..., 1] + x[..., 3] / 2) + padh
            labels[:, 1:] = y
            labels4.append(labels)
        labels4 = np.concatenate(labels4, 0)
        if d["mosaic"]:
            labels4[:, [1, 3]] = labels4[:, [1, 3]].clip(0, 2 * W)
            labels4[:, [2, 4]] = labels4[:, [2, 4]].clip(0, 2 * H)
        M, targets_ = np.asarray(d["M"], np.float64), labels4
        k = len(targets_)
        if not k:
            continue
        xy = np.ones((k * 4, 3))
        xy[:, :2] = targets_[:, [1, 2, 3, 4, 1, 4, 3, 2]].reshape(k * 4, 2)
        xy = xy @ M.T
        xy = (xy[:, :2] / xy[:, 2:3] if d["perspective"] else xy[:, :2]).reshape(k, 8)
        x, y = xy[:, [0, 2, 4, 6]], xy[:, [1, 3, 5, 7]]
        new = np.concatenate((x.min(1), y.min(1), x.max(1), y.max(1))).reshape(4, k).T
        new[:, [0, 2]] = new[:, [0, 2]].clip(0, W)
        new[:, [1, 3]] = new[:, [1, 3]].clip(0, H)
        i = box_candidates(box1=targets_[:, 1:5].T * d["s"], box2=new.T, area_thr=0.10)
        labels = targets_[i]
        labels[:, 1:5] = new[i]
        b = labels[:, 1:5]
        b[..., [0, 2]] = b[..., [0, 2]].clip(0, W - 1e-3)
        b[..., [1, 3]] = b[..., [1, 3]].clip(0, H - 1e-3)
        yy = np.copy(b)
        yy[..., 0] = ((b[..., 0] + b[..., 2]) / 2) / W
        yy[..., 1] = ((b[..., 1] + b[..., 3]) / 2) / H
        yy[..., 2] = (b[..., 2] - b[..., 0]) / W
        yy[..., 3] = (b[..., 3] - b[..., 1]) / H
        labels[:, 1:5] = yy
        if d["flip"]:
            labels[:, 1] = 1 - labels[:, 1]
        rows.append(np.concatenate([np.full((len(labels), 1), n, np.float32), labels], 1))
    return np.concatenate(rows) if rows else np.zeros((0, 6), np.float32)

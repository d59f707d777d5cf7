"""Batch-level, on-device form of the reference's img_aug (utils/datasets.py:63-68 -> contrast_and_brightness, :10-16).

The reference augments each uint8 HWC image on the host inside TensorDataset.__getitem__; with the input pipeline moved to the
GPU (uint8 batch copied first, `/255` fused into the stem) the same byte arithmetic runs on the whole uint8 batch in one
kernel of libyfv2.so (csrc/k_aug.cu), bit-identical to cv2.addWeighted.  (alpha, beta) are drawn per image from the same
random.uniform(0.25, 1.75) calls, in the same order as the reference would draw them image by image.

geometric_batch adds YOLOv5's geometric augmentation (load_mosaic, random_perspective, fliplr) before img_aug: the pixels in one
kernel pass (yfv2_engine.augment_geometric), the boxes moved alongside on the host (DESIGN.md §20)."""
import math
import random

import numpy as np
import torch

import yfv2_engine

HSV_GAINS = (0.0138, 0.678, 0.36)          # augment_hsv's defaults hgain, sgain, vgain (datasets.py:39)


def draw(n, H, W, rng=random, np_rng=np.random, *, motion_blur=False, random_resize=False, augment_hsv=False):
    """The per-image draws of img_aug (datasets.py:63-68) for n H x W images, in the reference's order: image by image alpha,
    beta; motion_blur's randint(1, 2) and, on 1, randint(2, 3) and uniform(-360, 360); rw, rh (all from `rng`); then the
    augment_hsv gains from `np_rng`.  Returns lists alpha, beta, blur (None or (degree, angle)), rw, rh, gains ([3] arrays);
    the lists of steps that are off stay empty."""
    alpha, beta, blur, rw, rh, gains = [], [], [], [], [], []
    for _ in range(n):
        alpha.append(rng.uniform(0.25, 1.75))
        beta.append(rng.uniform(0.25, 1.75))
        if motion_blur:
            blur.append((rng.randint(2, 3), rng.uniform(-360, 360)) if rng.randint(1, 2) == 1 else None)
        if random_resize:
            rw.append(int(W * rng.uniform(0.8, 1)))
            rh.append(int(H * rng.uniform(0.8, 1)))
        if augment_hsv:
            gains.append(np_rng.uniform(-1, 1, 3) * list(HSV_GAINS) + 1)
    return alpha, beta, blur, rw, rh, gains


def img_aug_batch(imgs_u8, rng=random, out=None, *, random_resize=False, augment_hsv=False, np_rng=np.random,
                  motion_blur=False):
    """imgs_u8: CUDA uint8 [N, ...] (any per-image layout).  Returns the augmented batch (new tensor unless `out` is given).

    random_resize / augment_hsv add the two steps img_aug lists after contrast_and_brightness (datasets.py:66-67, in that
    order; the batch must then be [N, 3, H, W] planar BGR).  Per image the draws follow the reference: alpha, beta, then
    rw = int(W * uniform(0.8, 1)) and rh = int(H * uniform(0.8, 1)) from `rng`, then the three augment_hsv gains from
    `np_rng`.  All steps run in one kernel pass (yfv2_engine.augment_batch).

    motion_blur adds img_aug's second step (datasets.py:65, :18-37): after beta each image draws randint(1, 2) from `rng`, and
    on 1 also degree = randint(2, 3) and angle = uniform(-360, 360); the blur then runs between contrast and the resize, in a
    first kernel pass over the blurred images."""
    n = imgs_u8.shape[0]
    if random_resize or augment_hsv or motion_blur:
        H, W = imgs_u8.shape[2], imgs_u8.shape[3]
        alpha, beta, blur, rw, rh, gains = draw(n, H, W, rng, np_rng, motion_blur=motion_blur, random_resize=random_resize,
                                                augment_hsv=augment_hsv)
        luts = yfv2_engine.hsv_luts(np.stack(gains)) if augment_hsv else None
        dst = out
        if random_resize and out is not None and out.data_ptr() == imgs_u8.data_ptr():
            dst = None                                                         # the resize reads neighbours: go through scratch
        res = yfv2_engine.augment_batch(imgs_u8, alpha, beta, rw if random_resize else None, rh if random_resize else None,
                                        luts, out=dst, blur=blur if motion_blur else None)
        if out is not None and res is not out:
            out.copy_(res)
            return out
        return res
    ab = [(rng.uniform(0.25, 1.75), rng.uniform(0.25, 1.75)) for _ in range(n)]      # alpha first, then beta (datasets.py:11-12)
    alpha = torch.tensor([a for a, _ in ab], dtype=torch.float32)
    beta = torch.tensor([b for _, b in ab], dtype=torch.float32)
    return yfv2_engine.contrast_and_brightness(imgs_u8, alpha, beta, out=out)


# YOLOv5's hyp.scratch-low values of the geometric hyperparameters
GEOM_HYP = dict(mosaic=1.0, degrees=0.0, translate=0.1, scale=0.5, shear=0.0, perspective=0.0, fliplr=0.5)


def _matmul3(a, b):
    """a @ b over stacks [n, 3, 3] of float64 matrices, each entry summed in index order, ((a_i0 b_0j + a_i1 b_1j) + a_i2 b_2j):
    elementwise numpy, no BLAS, so the bits are the same on every host."""
    return (a[:, :, 0, None] * b[:, None, 0, :] + a[:, :, 1, None] * b[:, None, 1, :]) + a[:, :, 2, None] * b[:, None, 2, :]


def draw_geometric(n, H, W, rng=random, *, mosaic=GEOM_HYP["mosaic"], degrees=GEOM_HYP["degrees"],
                   translate=GEOM_HYP["translate"], scale=GEOM_HYP["scale"], shear=GEOM_HYP["shear"],
                   perspective=GEOM_HYP["perspective"], fliplr=GEOM_HYP["fliplr"]):
    """The geometric draws of n H x W images, image by image from `rng`: random() < mosaic; with mosaic yc, xc =
    int(uniform(H // 2, 2H - H // 2)), int(uniform(W // 2, 2W - W // 2)), then choices(range(n), k=3) partners and a shuffle of
    [image] + partners (load_mosaic's lines, partners from the batch); random_perspective's eight draws in its order (perspective
    x, y, angle, scale, shear x, y, translate x, y); random() < fliplr.  Returns one dict per image: mosaic, xc, yc, src (the four
    tiles, or [image] * 4), M (float64 3x3, canvas -> output), s (the scale draw), perspective (whether cv2.warpPerspective runs:
    the hyperparameter is nonzero) and flip.  M = T @ S @ R @ P @ C as random_perspective builds it, associated as numpy evaluates
    that expression, ((((T @ S) @ R) @ P) @ C); the products are computed for all images at once (_matmul3)."""
    if n and mosaic > 0 and (H % 2 or W % 2):
        raise ValueError("mosaic needs even H and W (got %dx%d)" % (W, H))
    out = []
    mats = np.zeros((5, n, 3, 3))                                                # T, S, R, P, C of every image
    mats[:, :, [0, 1, 2], [0, 1, 2]] = 1.0
    T, S, R, P, C = mats
    for i in range(n):
        d = dict(mosaic=rng.random() < mosaic, xc=0, yc=0, src=[i] * 4)
        if d["mosaic"]:
            d["yc"] = int(rng.uniform(H // 2, 2 * H - H // 2))                   # mosaic_border (-H // 2, -W // 2)
            d["xc"] = int(rng.uniform(W // 2, 2 * W - W // 2))
            idx = [i] + rng.choices(range(n), k=3)
            rng.shuffle(idx)
            d["src"] = idx
        ch, cw = (2 * H, 2 * W) if d["mosaic"] else (H, W)                       # the canvas; the output is H x W either way
        C[i, 0, 2] = -cw / 2
        C[i, 1, 2] = -ch / 2
        P[i, 2, 0] = rng.uniform(-perspective, perspective)
        P[i, 2, 1] = rng.uniform(-perspective, perspective)
        a = rng.uniform(-degrees, degrees)
        s = rng.uniform(1 - scale, 1 + scale)
        ang = a * (math.pi / 180)                                                # cv2.getRotationMatrix2D(angle=a, center=(0, 0), s)
        alpha, beta = math.cos(ang) * s, math.sin(ang) * s
        R[i, 0, 0], R[i, 0, 1], R[i, 1, 0], R[i, 1, 1] = alpha, beta, -beta, alpha
        S[i, 0, 1] = math.tan(rng.uniform(-shear, shear) * math.pi / 180)
        S[i, 1, 0] = math.tan(rng.uniform(-shear, shear) * math.pi / 180)
        T[i, 0, 2] = rng.uniform(0.5 - translate, 0.5 + translate) * W
        T[i, 1, 2] = rng.uniform(0.5 - translate, 0.5 + translate) * H
        d["s"], d["perspective"] = s, bool(perspective)
        d["flip"] = rng.random() < fliplr
        out.append(d)
    M = _matmul3(_matmul3(_matmul3(_matmul3(T, S), R), P), C)
    for i, d in enumerate(out):
        d["M"] = M[i]
    return out


def geometric_targets(targets, draws, H, W):
    """The targets of draw_geometric's output images: rows (image, class, cx, cy, w, h) normalised, as the loaders produce them
    (CPU).  Per output image, YOLOv5's lines and dtypes: each tile's boxes to pixels by xywhn2xyxy in float32 (plus the tile's
    padw, padh), with mosaic clipped to [0, 2W] x [0, 2H]; random_perspective's corner transform and bounding box in float64
    (divided by the third coordinate with perspective), clipped to [0, W] x [0, H]; box_candidates(old * s, new, wh_thr=2,
    ar_thr=100, area_thr=0.10); back to float32 and xyxy2xywhn(clip=True, eps=1e-3); cx = 1 - cx on flip.  Rows come out image by
    image, in tile order, then in row order.  Returns a new float32 tensor (pinned when `targets` is).

    Every step is elementwise per row, so the rows of all tiles of all images are gathered once and each step runs over the whole
    batch, with each row's own padw, padh, M, s and flags: the same bits as the lines applied image by image."""
    t = targets.detach().cpu().numpy().astype(np.float32, copy=False) if isinstance(targets, torch.Tensor) else \
        np.asarray(targets, np.float32)
    n_out = len(draws)
    f32 = np.float32
    mosaic = np.array([bool(d["mosaic"]) for d in draws], bool)
    src = np.array([d["src"] for d in draws], np.int64).reshape(n_out, 4)
    xc = np.array([d["xc"] if d["mosaic"] else 0 for d in draws], np.int64)
    yc = np.array([d["yc"] if d["mosaic"] else 0 for d in draws], np.int64)
    M = np.array([np.asarray(d["M"], np.float64) for d in draws], np.float64).reshape(n_out, 3, 3)
    s = np.array([d["s"] for d in draws], np.float64)
    persp = np.array([bool(d["perspective"]) for d in draws], bool)
    flip = np.array([bool(d["flip"]) for d in draws], bool)

    # tiles in output order (image, then tile), and each tile's rows of t in row order
    tile_n, tile_k = np.nonzero(np.arange(4)[None, :] < np.where(mosaic, 4, 1)[:, None])
    tile_j = src[tile_n, tile_k]
    img = t[:, 0].astype(np.int64)
    order = np.argsort(img, kind="stable")
    first = np.searchsorted(img[order], tile_j, "left")
    count = np.searchsorted(img[order], tile_j, "right") - first
    rep = np.repeat(np.arange(len(tile_j)), count)
    within = np.arange(len(rep)) - np.repeat(np.cumsum(count) - count, count)
    lab = t[order[first[rep] + within]]
    n, k = tile_n[rep], tile_k[rep]
    mos = mosaic[n]
    padw = np.where(mos, xc[n] - np.where(k % 2 == 0, W, 0), 0).astype(f32)
    padh = np.where(mos, yc[n] - np.where(k < 2, H, 0), 0).astype(f32)
    x, y, w, h = lab[:, 2], lab[:, 3], lab[:, 4], lab[:, 5]
    b = np.stack([f32(W) * (x - w / f32(2)) + padw, f32(H) * (y - h / f32(2)) + padh,
                  f32(W) * (x + w / f32(2)) + padw, f32(H) * (y + h / f32(2)) + padh], 1).astype(np.float32)
    b[:, [0, 2]] = np.where(mos[:, None], b[:, [0, 2]].clip(0, 2 * W), b[:, [0, 2]])
    b[:, [1, 3]] = np.where(mos[:, None], b[:, [1, 3]].clip(0, 2 * H), b[:, [1, 3]])

    m = M[n]
    cx = b[:, [0, 2, 0, 2]].astype(np.float64)                                   # corners x1y1, x2y2, x1y2, x2y1
    cy = b[:, [1, 3, 3, 1]].astype(np.float64)
    X = cx * m[:, 0, 0, None] + cy * m[:, 0, 1, None] + m[:, 0, 2, None]
    Y = cx * m[:, 1, 0, None] + cy * m[:, 1, 1, None] + m[:, 1, 2, None]
    p = persp[n]
    if p.any():
        Z = cx[p] * m[p, 2, 0, None] + cy[p] * m[p, 2, 1, None] + m[p, 2, 2, None]
        X[p], Y[p] = X[p] / Z, Y[p] / Z
    new = np.stack([X.min(1), Y.min(1), X.max(1), Y.max(1)], 1)
    new[:, [0, 2]] = new[:, [0, 2]].clip(0, W)
    new[:, [1, 3]] = new[:, [1, 3]].clip(0, H)
    old = b * s[n].astype(np.float32)[:, None]                                   # float32, as box1=targets[:, 1:5].T * s
    w1, h1 = old[:, 2] - old[:, 0], old[:, 3] - old[:, 1]
    w2, h2 = new[:, 2] - new[:, 0], new[:, 3] - new[:, 1]
    ar = np.maximum(w2 / (h2 + 1e-16), h2 / (w2 + 1e-16))
    keep = (w2 > 2) & (h2 > 2) & (w2 * h2 / (w1 * h1 + 1e-16) > 0.10) & (ar < 100)
    xy = new[keep].astype(np.float32)
    xy[:, [0, 2]] = xy[:, [0, 2]].clip(0, W - 1e-3)                              # xyxy2xywhn(clip=True, eps=1e-3)
    xy[:, [1, 3]] = xy[:, [1, 3]].clip(0, H - 1e-3)
    r = np.zeros((len(xy), 6), np.float32)
    r[:, 0] = n[keep]
    r[:, 1] = lab[keep, 1]
    r[:, 2] = ((xy[:, 0] + xy[:, 2]) / 2) / W
    r[:, 3] = ((xy[:, 1] + xy[:, 3]) / 2) / H
    r[:, 4] = (xy[:, 2] - xy[:, 0]) / W
    r[:, 5] = (xy[:, 3] - xy[:, 1]) / H
    r[:, 2] = np.where(flip[n[keep]], 1 - r[:, 2], r[:, 2])
    res = torch.from_numpy(r)
    if isinstance(targets, torch.Tensor) and targets.is_pinned():
        res = res.pin_memory()
    return res


def geometric_batch(imgs_u8, targets, rng=random, out=None, **hyp):
    """YOLOv5's load_mosaic -> random_perspective -> fliplr on a CUDA uint8 [N, 3, H, W] batch and its CPU targets: the draws of
    draw_geometric (hyp: GEOM_HYP's keys, YOLOv5's hyp.scratch-low values by default), the pixels on the device in one pass
    (yfv2_engine.augment_geometric, into `out` when given; it must not overlap imgs_u8) and the targets on the host
    (geometric_targets).  Partners of a mosaic are drawn from the batch, and its tiles are the batch's W x H images.  Returns
    (images, targets)."""
    unknown = set(hyp) - set(GEOM_HYP)
    if unknown:
        raise TypeError("unknown geometric hyperparameters: %s" % ", ".join(sorted(unknown)))
    N, _, H, W = imgs_u8.shape
    draws = draw_geometric(N, H, W, rng, **hyp)
    imgs = yfv2_engine.augment_geometric(imgs_u8, draws, out=out)
    return imgs, geometric_targets(targets, draws, H, W)

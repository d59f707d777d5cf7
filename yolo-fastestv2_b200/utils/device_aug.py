"""Batch-level, on-device form of the reference's img_aug (utils/datasets.py:63-68 -> contrast_and_brightness, :10-16).

The reference augments each uint8 HWC image on the host inside TensorDataset.__getitem__; with the input pipeline moved to the
GPU (uint8 batch copied first, `/255` fused into the stem) the same byte arithmetic runs on the whole uint8 batch in one
kernel of libyfv2.so (csrc/k_aug.cu), bit-identical to cv2.addWeighted.  (alpha, beta) are drawn per image from the same
random.uniform(0.25, 1.75) calls, in the same order as the reference would draw them image by image."""
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

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


def img_aug_batch(imgs_u8, rng=random, out=None, *, random_resize=False, augment_hsv=False, np_rng=np.random):
    """imgs_u8: CUDA uint8 [N, ...] (any per-image layout).  Returns the augmented batch (new tensor unless `out` is given).

    random_resize / augment_hsv add the two steps img_aug lists after contrast_and_brightness (datasets.py:66-67, in that
    order; the batch must then be [N, 3, H, W] planar BGR).  Per image the draws follow the reference: alpha, beta, then
    rw = int(W * uniform(0.8, 1)) and rh = int(H * uniform(0.8, 1)) from `rng`, then the three augment_hsv gains from
    `np_rng`.  All steps run in one kernel pass (yfv2_engine.augment_batch)."""
    n = imgs_u8.shape[0]
    if random_resize or augment_hsv:
        H, W = imgs_u8.shape[2], imgs_u8.shape[3]
        alpha, beta, rw, rh, gains = [], [], [], [], []
        for _ in range(n):
            alpha.append(rng.uniform(0.25, 1.75))
            beta.append(rng.uniform(0.25, 1.75))
            if random_resize:
                rw.append(int(W * rng.uniform(0.8, 1)))
                rh.append(int(H * rng.uniform(0.8, 1)))
            if augment_hsv:
                gains.append(np_rng.uniform(-1, 1, 3) * list(HSV_GAINS) + 1)
        luts = yfv2_engine.hsv_luts(np.stack(gains)) if augment_hsv else None
        dst = out
        if random_resize and out is not None and out.data_ptr() == imgs_u8.data_ptr():
            dst = None                                                         # the resize reads neighbours: go through scratch
        res = yfv2_engine.augment_batch(imgs_u8, alpha, beta, rw if random_resize else None, rh if random_resize else None,
                                        luts, out=dst)
        if out is not None and res is not out:
            out.copy_(res)
            return out
        return res
    ab = [(rng.uniform(0.25, 1.75), rng.uniform(0.25, 1.75)) for _ in range(n)]      # alpha first, then beta (datasets.py:11-12)
    alpha = torch.tensor([a for a, _ in ab], dtype=torch.float32)
    beta = torch.tensor([b for _, b in ab], dtype=torch.float32)
    return yfv2_engine.contrast_and_brightness(imgs_u8, alpha, beta, out=out)

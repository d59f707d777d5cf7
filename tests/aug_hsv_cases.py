"""Seeded inputs of tests/golden/aug_hsv_cases.npz (tests/golden/make_golden_aug_hsv.py) and the tests that read it."""
import numpy as np


def image(seed, h, w):
    return np.random.RandomState(seed).randint(0, 256, (h, w, 3)).astype(np.uint8)


# augment_hsv: (name, image, u) with r = u * (hgain, sgain, vgain) + 1.  u = 0 is the identity LUT; +-1 are both ends of each
# gain; u0 = 1 (r0 = 1.0138) wraps hue 178 and 179 past 180; u1, u2 > 0 clip saturation and value at 255.
HSV_CASES = [
    ("identity", (1, 352, 352), (0.0, 0.0, 0.0)),
    ("max", (2, 352, 352), (1.0, 1.0, 1.0)),
    ("min", (3, 352, 352), (-1.0, -1.0, -1.0)),
    ("mixed_a", (4, 37, 53), (1.0, -1.0, 1.0)),
    ("mixed_b", (5, 37, 53), (-1.0, 1.0, -1.0)),
    ("row", (6, 1, 97), (0.7, 0.9, 0.95)),
    ("col", (7, 89, 1), (-0.3, 0.5, 1.0)),
    ("draw_a", (8, 352, 352), (0.4055, -0.21, 0.77)),
    ("draw_b", (9, 37, 53), (-0.62, 0.33, -0.48)),
]

# random_resize: (name, image, (rw, rh))
RESIZE_CASES = [
    ("281x281", (11, 352, 352), (281, 281)),
    ("282x351", (12, 352, 352), (282, 351)),
    ("351x282", (13, 352, 352), (351, 282)),
    ("352x352", (14, 352, 352), (352, 352)),
    ("odd", (15, 37, 53), (43, 30)),
]
RESIZE_SEEDS = (0, 1, 2)

# the full chain: per seed a batch of CHAIN_N 352 x 352 images
CHAIN_SEEDS = (0, 1, 7)
CHAIN_N = 3


def chain_batch(seed):
    return [image(100 + 10 * seed + i, 352, 352) for i in range(CHAIN_N)]

"""Generates tests/golden/stem.npz: the stem output (conv3x3/2 + BN + ReLU + maxpool3x3/2, debug_gather tap 0) for uint8 and
fp32 inputs, as the kernel computed it while the uint8 input was still staged by synchronous uchar4 loads converted with
__fdiv_rn.  The asynchronous staging that replaced them must reproduce it bit for bit.  Frozen on an H100 with that build:

    python tests/golden/make_golden_stem.py [OUT.npz]

Per shape `<h>x<w>` (one image; state dict and images seeded by the shape) and input `u8` / `f32`: the [1, 24, h/4, w/4] tap
itself for the small shapes, `<h>x<w>_<input>_sha256` (SHA-256 of the float32 tap bytes) for the large ones.
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (os.path.dirname(os.path.dirname(HERE)), os.path.dirname(HERE)):    # the repository and tests/
    sys.path.insert(0, p)

# 640x640 runs 4 column tiles of 40 pooled columns; 96x416 runs 3 tiles, the last one narrower (35, 35, 34); 352x352 and
# 96x128 end in a shorter band; 32x32 is one item
SHAPES = [(352, 352), (640, 640), (96, 416), (96, 128), (64, 96), (32, 32)]
DIGEST_ONLY = {(352, 352), (640, 640), (96, 416)}


def seeds(h, w):
    return 900 + h + w, 1000 + h + w


def make_model(sd_seed):
    import yfv2  # noqa: F401
    import model.detector as det
    import synth
    m = det.Detector(80, 3, True)
    m.load_state_dict(synth.make_state_dict(sd_seed), strict=True)
    return m.cuda().eval()


def make_inputs(seed, n, h, w):
    """uint8 images (every byte value) and fp32 images in [0, 1), on the host."""
    import torch
    import synth
    rs = np.random.RandomState(seed)
    u8 = torch.from_numpy(rs.randint(0, 256, size=(n, 3, h, w), dtype=np.uint8))
    return {"u8": u8, "f32": synth.make_images(seed + 1, n, h, w)}


def stem_tap(m, x):
    """The stem output of x (CUDA, uint8 or fp32, any alignment) after running the stem launch alone."""
    plan = m._plan_for(x)
    preds = plan.alloc_preds()
    plan.forward_range(x, preds, 0, 1)
    return plan.debug_gather(0).cpu().numpy()


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.float32).tobytes()).hexdigest()


def stem_taps(h, w):
    sd_seed, x_seed = seeds(h, w)
    m = make_model(sd_seed)
    return {k: stem_tap(m, x.cuda()) for k, x in make_inputs(x_seed, 1, h, w).items()}


if __name__ == "__main__":
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "stem.npz")
    arrays = {}
    for h, w in SHAPES:
        for k, v in stem_taps(h, w).items():
            if (h, w) in DIGEST_ONLY:
                arrays["%dx%d_%s_sha256" % (h, w, k)] = np.array(digest(v))
            else:
                arrays["%dx%d_%s" % (h, w, k)] = v
    np.savez_compressed(path, **arrays)
    print("wrote", path, sorted(arrays))

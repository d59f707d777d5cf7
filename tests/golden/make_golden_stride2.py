"""Generates tests/golden/stride2_banded.npz: digests of the outputs of the stride-2 blocks stage2.0 and stage3.0 as
blk_kernel<K, 2> computes them, so that the band walk that replaced it (walk::blk_kernel<K, 2> in k_net.cu) can be pinned to it
bit for bit.  Frozen on an H100 (132 SMs) with the build before the band walk existed:

    python tests/golden/make_golden_stride2.py [OUT.npz]

Per shape `<n>x<h>x<w>` (state dict and images seeded by the shape): `<n>x<h>x<w>_stage2.0_<i>` and `<n>x<h>x<w>_stage3.0_<i>`,
the SHA-256 (hex) of the block output of image i, as little-endian float32 in the reference's logical channel order
(debug_gather, [C, H, W]), after running the forward one fused stage at a time.  A digest pins every bit at a few hundred bytes
per tap; the outputs themselves (0.56 MB per 352^2 image) would make the file several megabytes.  The shapes reach, at 132 SMs:
  64x352x352  multi-row bands with a shorter last band (stage2.0 R = 5 of 44 rows, stage3.0 R = 4 of 22), images 0 and 63
  1x352x352   one-row bands
  2x64x96     stage2.0 input 24 columns wide, so 16-pixel tiles straddle rows
  1x32x32     the smallest maps (stage3.0: 4x4 -> 2x2)
  1x640x640
  1x64x1024   stage3.0 (128 input columns) past the shared memory of the band walk: the one-pass blk_kernel<48, 2> runs it
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (os.path.dirname(os.path.dirname(HERE)), os.path.dirname(HERE)):    # the repository and tests/
    sys.path.insert(0, p)

SHAPES = [(64, 352, 352, (0, 63)), (1, 352, 352, (0,)), (2, 64, 96, (0, 1)), (1, 32, 32, (0,)), (1, 640, 640, (0,)),
          (1, 64, 1024, (0,))]
TAP = {"stage2.0": 1, "stage3.0": 5}


def seeds(n, h, w):
    return 900 + n + h + w, 1000 + n + h + w


def digest(a):
    """SHA-256 (hex) of an array as contiguous little-endian float32."""
    return hashlib.sha256(np.ascontiguousarray(a, dtype="<f4").tobytes()).hexdigest()


def make_model(sd):
    import model.detector as det
    m = det.Detector(80, 3, True)
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()


def stride2_taps(n, h, w, images):
    """{"stage2.0": [len(images), 48, h/8, w/8], "stage3.0": [len(images), 96, h/16, w/16]} after a forward run one fused stage
    at a time."""
    import torch
    import yfv2  # noqa: F401
    import synth
    sd_seed, x_seed = seeds(n, h, w)
    m = make_model(synth.make_state_dict(sd_seed))
    x = synth.make_images(x_seed, n, h, w).cuda()
    preds = m(x)
    plan = next(iter(m._plans.values()))
    names = plan.stage_names
    out = {}
    for i in range(names.index("stage3.0") + 1):
        plan.forward_range(x, preds, i, i + 1)
        if names[i] in TAP:
            out[names[i]] = plan.debug_gather(TAP[names[i]])[list(images)].cpu().numpy()
    torch.cuda.synchronize()
    return out


if __name__ == "__main__":
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "stride2_banded.npz")
    arrays = {}
    for n, h, w, images in SHAPES:
        for k, v in stride2_taps(n, h, w, images).items():
            for j, i in enumerate(images):
                arrays["%dx%dx%d_%s_%d" % (n, h, w, k, i)] = np.array(digest(v[j]))
    np.savez_compressed(path, **arrays)
    print("wrote", path, sorted(arrays))

"""Generates tests/golden/stride1_banded.npz: digests of the outputs of the single stride-1 blocks of stages 2 and 3 (stage2.1-3,
K = 24; stage3.1-7, K = 48) as blk_kernel<K, 1> computes them, so that the band walk that replaced it (walk::blk_kernel<K, 1> in
k_net.cu) can be pinned to it bit for bit.  Frozen on an H100 (132 SMs) with the build before the stride-1 band walk existed:

    python tests/golden/make_golden_stride1.py [OUT.npz]

Per shape `<n>x<h>x<w>` (state dict and images seeded by the shape): `<n>x<h>x<w>_<stage>_<i>` for each stage2.1-3 and
stage3.1-7, the SHA-256 (hex) of the block output of image i, as little-endian float32 in the reference's logical channel order
(debug_gather, [C, H, W]), after running the forward one fused stage at a time.  The shapes reach, at 132 SMs:
  256x352x352  stage2.x R = 22 (two equal bands), stage3.x R = 17 with a 5-row last band; images 0, 1, 254 and 255
  64x352x352   stage2.x R = 6 of 44 rows, stage3.x R = 5 of 22: both with a shorter last band
  1x352x352    one-row bands
  1x640x640
  1x128x1024   stage2.x at 128 columns on the walk, stage3.x at 64 columns past its shared memory
  1x128x1280   stage2.x at 160 columns and stage3.x at 80: both past the walk
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (os.path.dirname(os.path.dirname(HERE)), os.path.dirname(HERE)):    # the repository and tests/
    sys.path.insert(0, p)

SHAPES = [(256, 352, 352, (0, 1, 254, 255)), (64, 352, 352, (0, 63)), (1, 352, 352, (0,)), (1, 640, 640, (0,)),
          (1, 128, 1024, (0,)), (1, 128, 1280, (0,))]
TAP = dict([("stage2.%d" % j, 1 + j) for j in (1, 2, 3)] + [("stage3.%d" % j, 5 + j) for j in range(1, 8)])


def seeds(n, h, w):
    return 1100 + n + h + w, 1200 + n + h + w


def digest(a):
    """SHA-256 (hex) of an array as contiguous little-endian float32."""
    return hashlib.sha256(np.ascontiguousarray(a, dtype="<f4").tobytes()).hexdigest()


def make_model(sd):
    import model.detector as det
    m = det.Detector(80, 3, True)
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()


def stride1_taps(m, x, images=None):
    """{stage: [images, C, H, W]} of every stage2.1-3 and stage3.1-7 block output of the batch x (m holds this one plan), after a
    forward run one fused stage at a time up to stage3.7."""
    import torch
    preds = m(x)
    plan = next(iter(m._plans.values()))
    names = plan.stage_names
    out = {}
    for i in range(names.index("stage3.7") + 1):
        plan.forward_range(x, preds, i, i + 1)
        if names[i] in TAP:
            v = plan.debug_gather(TAP[names[i]])
            out[names[i]] = (v if images is None else v[list(images)]).cpu().numpy()
    torch.cuda.synchronize()
    return out


def shape_taps(n, h, w, images):
    import yfv2  # noqa: F401
    import synth
    sd_seed, x_seed = seeds(n, h, w)
    return stride1_taps(make_model(synth.make_state_dict(sd_seed)), synth.make_images(x_seed, n, h, w).cuda(), images)


if __name__ == "__main__":
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "stride1_banded.npz")
    arrays = {}
    for n, h, w, images in SHAPES:
        for k, v in shape_taps(n, h, w, images).items():
            for j, i in enumerate(images):
                arrays["%dx%dx%d_%s_%d" % (n, h, w, k, i)] = np.array(digest(v[j]))
    np.savez_compressed(path, **arrays)
    print("wrote", path, len(arrays), "digests")

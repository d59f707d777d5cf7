"""Generates tests/golden/stage4_banded.npz: the outputs of backbone stage 4 as the banded block kernel computes them, so that
the whole-image kernels (the K = 96 stride-2 block on whole images and the one-CTA-per-SM stride-1 chain) can be pinned to it
bit for bit at the shapes where they replace it.  Frozen on an H100 with the build before those kernels existed, where stage4.0
ran blk_kernel<96, 2> in 1-row bands and stage4.1-3 ran as three banded launches at every shape:

    python tests/golden/make_golden_stage4.py [OUT.npz]

Per shape `<h>x<w>` (one image, state dict and image seeded by the shape): `<h>x<w>_stage4.0` and `<h>x<w>_stage4.3`, the
block outputs in the reference's logical channel order (debug_gather), each after running the forward one fused stage at a time.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (os.path.dirname(os.path.dirname(HERE)), os.path.dirname(HERE)):    # the repository and tests/
    sys.path.insert(0, p)

SHAPES = [(352, 352), (224, 96)]
TAP = {"stage4.0": 13, "stage4.3": 16}


def seeds(h, w):
    return 700 + h + w, 800 + h + w


def stage4_taps(h, w):
    """Taps of stage4.0 and stage4.3 after a forward run one fused stage at a time (what the suite does with the current build)."""
    import torch
    import yfv2  # noqa: F401
    import synth
    import model.detector as det
    sd_seed, x_seed = seeds(h, w)
    m = det.Detector(80, 3, True)
    m.load_state_dict(synth.make_state_dict(sd_seed), strict=True)
    m = m.cuda().eval()
    x = synth.make_images(x_seed, 1, h, w).cuda()
    preds = m(x)
    plan = next(iter(m._plans.values()))
    names = plan.stage_names
    out = {}
    for i in range(len(names)):
        plan.forward_range(x, preds, i, i + 1)
        if names[i] in TAP:
            out[names[i]] = plan.debug_gather(TAP[names[i]]).cpu().numpy()
    torch.cuda.synchronize()
    return out


if __name__ == "__main__":
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "stage4_banded.npz")
    arrays = {}
    for h, w in SHAPES:
        for k, v in stage4_taps(h, w).items():
            arrays["%dx%d_%s" % (h, w, k)] = v
    np.savez_compressed(path, **arrays)
    print("wrote", path, sorted(arrays))

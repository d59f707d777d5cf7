"""Generates tests/golden/heads.npz: digests of what the four head launches (head_kernel<0>, head_kernel<1>, head2_kernel in
k_net.cu) compute, so that the staged-window A operand that replaced their global-load stencils can be pinned to them bit for bit.
Frozen on an H100 (132 SMs) with the build before the heads staged their input windows in shared memory:

    python tests/golden/make_golden_heads.py [OUT.npz]

Per shape `<n>x<h>x<w>_a<A>c<C>` (state dict and images seeded by the shape): `..._tap<t>_<i>` for the heads.a outputs (debug_gather
taps 19-22: cls2, reg2, cls3, reg3 mid-head planes) and `..._pred<k>_<i>` for the six head tensors (reg2, obj2, cls2, reg3, obj3,
cls3), the SHA-256 (hex) of image i as little-endian float32, after running the forward one fused stage at a time.  The shapes:
  64x352x352    22x22 and 11x11 maps: 128-pixel chunks straddle rows and the last chunk at 22x22 is short (100 pixels)
  1x32x32       2x2 and 1x1 maps: most warps of a CTA hold no pixel
  1x640x32      one-pixel-wide map (40x2, 20x1)
  1x32x640      one-pixel-tall map (2x40, 1x20)
  1x640x640     40x40 and 20x20
  2x96x128      150 classes: head2_kernel
  2x128x128     A = 2, C = 20
  1x32x2560     2x160: an 8-channel window of 6 rows of 164 floats does not fit three times next to the weights with two CTAs per
                SM, so heads2.a and heads2.b take the global-load path (1x80 at stride 32 is staged)
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (os.path.dirname(os.path.dirname(HERE)), os.path.dirname(HERE)):    # the repository and tests/
    sys.path.insert(0, p)

# (n, h, w, A, C, images whose digests are kept)
SHAPES = [(64, 352, 352, 3, 80, (0, 63)), (1, 32, 32, 3, 80, (0,)), (1, 640, 32, 3, 80, (0,)), (1, 32, 640, 3, 80, (0,)),
          (1, 640, 640, 3, 80, (0,)), (2, 96, 128, 3, 150, (0, 1)), (2, 128, 128, 2, 20, (0, 1)), (1, 32, 2560, 3, 80, (0,))]
TAPS = (19, 20, 21, 22)


def key(n, h, w, a, c):
    return "%dx%dx%d_a%dc%d" % (n, h, w, a, c)


def seeds(n, h, w, a, c):
    return 1300 + n + h + w + a + c, 1400 + n + h + w + a + c


def digest(a):
    """SHA-256 (hex) of an array as contiguous little-endian float32."""
    return hashlib.sha256(np.ascontiguousarray(a, dtype="<f4").tobytes()).hexdigest()


def make_model(sd, a, c):
    import model.detector as det
    m = det.Detector(c, a, True)
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()


def run_stages(m, x):
    """({tap: [N, 72, h, w]}, [six head tensors]) of the batch x (m holds this one plan), after running the forward one fused stage
    at a time."""
    import torch
    preds = m(x)
    plan = next(iter(m._plans.values()))
    for i in range(len(plan.stage_names)):
        plan.forward_range(x, preds, i, i + 1)
    taps = {t: plan.debug_gather(t).cpu().numpy() for t in TAPS}
    torch.cuda.synchronize()
    return taps, [p.cpu().numpy() for p in preds]


def head_outputs(n, h, w, a, c):
    import yfv2  # noqa: F401
    import synth
    sd_seed, x_seed = seeds(n, h, w, a, c)
    m = make_model(synth.make_state_dict(sd_seed, classes=c, anchor_num=a), a, c)
    return run_stages(m, synth.make_images(x_seed, n, h, w).cuda())


def digests(n, h, w, a, c, images):
    taps, preds = head_outputs(n, h, w, a, c)
    out = {}
    for i in images:
        for t in TAPS:
            out["%s_tap%d_%d" % (key(n, h, w, a, c), t, i)] = digest(taps[t][i])
        for k, p in enumerate(preds):
            out["%s_pred%d_%d" % (key(n, h, w, a, c), k, i)] = digest(p[i])
    return out


if __name__ == "__main__":
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "heads.npz")
    arrays = {}
    for n, h, w, a, c, images in SHAPES:
        arrays.update({k: np.array(v) for k, v in digests(n, h, w, a, c, images).items()})
    np.savez_compressed(path, **arrays)
    print("wrote", path, len(arrays), "digests")

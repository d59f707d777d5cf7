"""The stem launch (conv3x3/2 + BN + ReLU + maxpool3x3/2, debug_gather tap 0) bit for bit: against tests/golden/stem.npz, which
froze it before the uint8 patch was staged asynchronously, and image for image between a batch and the same images run
alone.  One image gives at most one item per CTA (352x352: 36 items on 36 CTAs), so the batches are sized to give every CTA
several items, the case where the next item's pixels are fetched while the current one convolves.  Each check also runs an
uint8 view whose base is not 4-byte aligned, which takes the scalar loads."""
import importlib.util
import os

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401

pytestmark = pytest.mark.gpu

_spec = importlib.util.spec_from_file_location(
    "make_golden_stem", os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_golden_stem.py"))
mk = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mk)


def unaligned(x):
    """x (uint8) copied into a CUDA view whose base is one byte past an allocation's start."""
    buf = torch.empty(x.numel() + 1, dtype=torch.uint8, device="cuda")
    v = buf[1:].view(x.shape)
    v.copy_(x)
    assert v.data_ptr() % 4 != 0 and v.is_contiguous()
    return v


@pytest.mark.parametrize("h,w", mk.SHAPES)
def test_stem_matches_golden(golden_dir, h, w):
    g = np.load(os.path.join(golden_dir, "stem.npz"))
    sd_seed, x_seed = mk.seeds(h, w)
    m = mk.make_model(sd_seed)
    xs = mk.make_inputs(x_seed, 1, h, w)
    got = {k: mk.stem_tap(m, x.cuda()) for k, x in xs.items()}
    got["u8_unaligned"] = mk.stem_tap(m, unaligned(xs["u8"]))
    for k, v in got.items():
        key = "%dx%d_%s" % (h, w, k.split("_")[0])
        if (h, w) in mk.DIGEST_ONLY:
            assert mk.digest(v) == str(g[key + "_sha256"]), k
        else:
            assert np.array_equal(v, g[key]), k


@pytest.mark.parametrize("n,h,w", [(16, 352, 352), (300, 64, 64)])
def test_batch_equals_images_alone(n, h, w):
    m = mk.make_model(77)
    xs = mk.make_inputs(78, n, h, w)
    for k, x in xs.items():
        x = x.cuda()
        alone = [mk.stem_tap(m, x[i:i + 1])[0] for i in range(n)]
        bigs = {k: mk.stem_tap(m, x)}
        if k == "u8":
            bigs["u8_unaligned"] = mk.stem_tap(m, unaligned(xs["u8"]))
        for kb, big in bigs.items():
            for i in range(n):
                assert np.array_equal(big[i], alone[i]), (kb, i)

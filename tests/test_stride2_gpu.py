"""The stride-2 blocks stage2.0 (K = 24) and stage3.0 (K = 48) on the band walk (walk::blk_kernel<K, 2>): bit for bit what the
one-pass blk_kernel<K, 2> computed (digests in tests/golden/stride2_banded.npz), on the band walk where it fits and on the
one-pass kernel where it does not, and batch-invariant across the band and image boundaries of the walk."""
import importlib.util
import os

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import net_dispatch as nd
import synth

pytestmark = pytest.mark.gpu
TAP = {"stage2.0": 1, "stage3.0": 5}


def golden_module(golden_dir):
    spec = importlib.util.spec_from_file_location("make_golden_stride2", os.path.join(golden_dir, "make_golden_stride2.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    return mk


def taps(m, x):
    """Taps of stage2.0 and stage3.0 of the batch x (m holds this one plan), after running the forward one fused stage at a time
    up to stage3.0."""
    preds = m(x)
    plan = next(iter(m._plans.values()))
    names = plan.stage_names
    out = {}
    for i in range(names.index("stage3.0") + 1):
        plan.forward_range(x, preds, i, i + 1)
        if names[i] in TAP:
            out[names[i]] = plan.debug_gather(TAP[names[i]]).cpu().numpy()
    return out


def profiled_kernel_names(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {e.name.replace(" ", "") for e in prof.events()}


# k_net.cu walk::smem_bytes and blk_s2_walk_fits, for the plan's pool planes (one-pixel frame, rows of align4(W + 2) floats)
def walk_smem_bytes(k, wi):
    ws = (wi + 2 + 3) // 4 * 4
    cs = 5 * ws                                  # ring of 4 G + 1 rows, G = 1
    while cs % 32 not in (8, 24):
        cs += 4
    return (3 * (k * nd.w_stride(k) + 2 * k) + 24 * k + k * cs + k * 3 * (wi + 2)) * 4


def walk_fits(k, wi):
    return k in (24, 48) and walk_smem_bytes(k, wi) <= nd.K_SMEM_CAP


SHAPES = [(n, h, w) for n, h, w, _ in golden_module(os.path.join(os.path.dirname(__file__), "golden")).SHAPES]


@pytest.mark.parametrize("n,h,w", SHAPES)
def test_matches_the_banded_kernel(golden_dir, n, h, w):
    mk = golden_module(golden_dir)
    images = dict(((s[0], s[1], s[2]), s[3]) for s in mk.SHAPES)[(n, h, w)]
    g = np.load(os.path.join(golden_dir, "stride2_banded.npz"))
    got = mk.stride2_taps(n, h, w, images)
    for k, v in got.items():
        for j, i in enumerate(images):
            assert mk.digest(v[j]) == str(g["%dx%dx%d_%s_%d" % (n, h, w, k, i)]), (k, i)


def test_selection_at_the_fit_boundary():
    """The band walk fits up to 286 input columns at K = 24 (stage2.0) and up to 122 at K = 48 (stage3.0), so stage3.0 leaves it
    between 960 and 992 image columns while stage2.0 stays on it.  Both kernels are blk_kernel<K, 2>, one CTA per band; the walk is
    the one in namespace walk."""
    assert walk_fits(24, 286) and not walk_fits(24, 287)
    assert walk_fits(48, 122) and not walk_fits(48, 123)
    assert walk_smem_bytes(24, 88) <= 113 * 1024 and walk_smem_bytes(48, 44) <= 113 * 1024      # 352^2: two CTAs per SM
    want = {960: {"walk::blk_kernel<24,2>", "walk::blk_kernel<48,2>"},
            1024: {"walk::blk_kernel<24,2>", "namespace)::blk_kernel<48,2>"}}
    m = golden_module(os.path.join(os.path.dirname(__file__), "golden")).make_model(synth.make_state_dict(11))
    for w, kerns in want.items():
        x = synth.make_images(12, 1, 64, w).cuda()
        m(x)
        names = profiled_kernel_names(lambda: [m(x) for _ in range(3)])     # a record at the edge of a trace can be lost
        ran = {k for k in ("walk::blk_kernel<24,2>", "walk::blk_kernel<48,2>", "namespace)::blk_kernel<24,2>",
                           "namespace)::blk_kernel<48,2>") if any(k + "(" in e for e in names)}
        assert ran == kerns, (w, ran)


@pytest.mark.parametrize("n,h,w", [(256, 352, 352), (50, 352, 352), (300, 32, 32)])
def test_batch_equals_images_alone(n, h, w):
    """At 256 and 50 x 352^2 stage2.0 runs 5-row bands with a shorter last one (R = 5 of 44 rows) and stage3.0 R = 4 of 22; at
    300 x 32^2 one band per image.  Every image equals, bit for bit, the same image run alone (one-row bands at 352^2): no row
    carried from one step to the next leaks across a band or an image."""
    mk = golden_module(os.path.join(os.path.dirname(__file__), "golden"))
    sd = synth.make_state_dict(81)
    x = synth.make_images(82, n, h, w).cuda()
    big = taps(mk.make_model(sd), x)
    m1 = mk.make_model(sd)                # one plan, batch 1
    for i in range(n):
        one = taps(m1, x[i:i + 1])
        for k in TAP:
            assert np.array_equal(big[k][i], one[k][0]), (k, i)

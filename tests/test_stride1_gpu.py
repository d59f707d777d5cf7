"""The single stride-1 blocks of stages 2 and 3 (stage2.1-3, K = 24; stage3.1-7, K = 48) on the band walk
(walk::blk_kernel<K, 1>): bit for bit what blk_kernel<K, 1> computed (digests in tests/golden/stride1_banded.npz), on the walk
where it fits and on blk_kernel<K, 1> where it does not, and batch-invariant across the bands and images a CTA walks in turn."""
import importlib.util
import os

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import net_dispatch as nd
import synth

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def golden_module():
    spec = importlib.util.spec_from_file_location("make_golden_stride1", os.path.join(GOLDEN, "make_golden_stride1.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    return mk


def profiled_kernel_names(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {e.name.replace(" ", "") for e in prof.events()}


# k_net.cu walk::s1_smem_bytes and blk_s1_walk_step, for the plan's pool planes (one-pixel frame, rows of align4(W + 2) floats)
S1_STEP_MAX = {24: 4, 48: 3}
S1_WALK_BUDGET = 113 * 1024


def walk_smem_bytes(k, g, wi):
    ws = (wi + 2 + 3) // 4 * 4
    cs = (2 * g + 2) * ws
    while cs % 32 not in (8, 24):
        cs += 4
    return (2 * (k * nd.w_stride(k) + 2 * k) + 12 * k + k * cs + k * (g + 2) * (wi + 2)) * 4


def walk_step(k, wi):
    if k not in (24, 48):
        return 0
    return next((g for g in range(S1_STEP_MAX[k], 0, -1) if walk_smem_bytes(k, g, wi) <= S1_WALK_BUDGET), 0)


def stride1_launches(n, h, w):
    return [L for L in nd.launches(n, h, w) if L.site in ("stage2.s1", "stage3.s1")]


MK = golden_module()
SHAPES = [(n, h, w) for n, h, w, _ in MK.SHAPES]


def test_shapes_reach_their_cells():
    """Each golden shape reaches the band layout and the side of the fit rule it was chosen for, at 132 SMs."""
    want = {(256, 352, 352): {"stage2": (22, False), "stage3": (17, True)},
            (64, 352, 352): {"stage2": (6, True), "stage3": (5, True)},
            (1, 352, 352): {"stage2": (1, False), "stage3": (1, False)}}
    for n, h, w in SHAPES:
        ls = stride1_launches(n, h, w)
        assert len(ls) == 10 and all(L.variant != "chain" for L in ls), (n, h, w)
        for L in ls:
            stage = L.site.split(".")[0]
            if (n, h, w) in want:
                assert (L.R, L.partial) == want[(n, h, w)][stage], (n, h, w, L)
    assert walk_step(24, 1024 // 8) >= 1 and walk_step(48, 1024 // 16) == 0   # 1x128x1024: stage2 on the walk, stage3 past it
    assert walk_step(24, 1280 // 8) == 0 and walk_step(48, 1280 // 16) == 0   # 1x128x1280: both past it


@pytest.mark.parametrize("n,h,w", SHAPES)
def test_matches_blk_kernel(n, h, w):
    images = dict(((s[0], s[1], s[2]), s[3]) for s in MK.SHAPES)[(n, h, w)]
    g = np.load(os.path.join(GOLDEN, "stride1_banded.npz"))
    got = MK.shape_taps(n, h, w, images)
    assert sorted(got) == sorted(MK.TAP)
    for k, v in got.items():
        for j, i in enumerate(images):
            assert MK.digest(v[j]) == str(g["%dx%dx%d_%s_%d" % (n, h, w, k, i)]), (k, i)


def test_selection_at_the_fit_boundary():
    """The walk fits up to 158 columns at K = 24 and up to 62 at K = 48 (one-row steps); at 352^2 it keeps two CTAs per SM with
    steps of 4 rows at K = 24 and 3 at K = 48.  Past the boundary blk_kernel<K, 1> (anonymous namespace) runs the block."""
    assert walk_step(24, 158) == 1 and walk_step(24, 159) == 0
    assert walk_step(48, 62) == 1 and walk_step(48, 63) == 0
    assert walk_step(24, 44) == 4 and walk_step(48, 22) == 3
    want = {1024: {"walk::blk_kernel<24,1>", "namespace)::blk_kernel<48,1>"},
            1280: {"namespace)::blk_kernel<24,1>", "namespace)::blk_kernel<48,1>"},
            960: {"walk::blk_kernel<24,1>", "walk::blk_kernel<48,1>"}}
    m = MK.make_model(synth.make_state_dict(11))
    for w, kerns in want.items():
        x = synth.make_images(12, 1, 128, w).cuda()
        m(x)
        names = profiled_kernel_names(lambda: [m(x) for _ in range(3)])     # a record at the edge of a trace can be lost
        ran = {k for k in ("walk::blk_kernel<24,1>", "walk::blk_kernel<48,1>", "namespace)::blk_kernel<24,1>",
                           "namespace)::blk_kernel<48,1>") if any(k + "(" in e for e in names)}
        assert ran == kerns, (w, ran)


@pytest.mark.parametrize("n,h,w", [(256, 352, 352), (50, 352, 352), (300, 320, 320)])
def test_batch_equals_images_alone(n, h, w):
    """Banded launches with several items per CTA: at 256 x 352^2 stage3.x runs 17- and 5-row bands, at 50 x 352^2 R = 6 / 3
    with shorter last bands, at 300 x 320^2 600 items with shorter last bands in both stages.  Every image equals, bit for bit,
    the same image run alone (one-row bands): neither the rows a CTA stages ahead for its next item nor the order in which it
    takes its items leaks anything between bands or images."""
    for L in stride1_launches(n, h, w):
        assert L.R > 1 and L.items > 264, L
    sd = synth.make_state_dict(91)
    x = synth.make_images(92, n, h, w).cuda()
    big = MK.stride1_taps(MK.make_model(sd), x)
    m1 = MK.make_model(sd)                # one plan, batch 1
    for i in range(n):
        one = MK.stride1_taps(m1, x[i:i + 1])
        for k in MK.TAP:
            assert np.array_equal(big[k][i], one[k][0]), (k, i)

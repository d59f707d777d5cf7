"""The four head launches (head_kernel<0>, head_kernel<1>, head2_kernel) with their 5x5 depthwise taps read from windows staged in
shared memory: bit for bit what the global-load stencils computed (digests in tests/golden/heads.npz), on the staged path where it
fits and on the plane reads where it does not, and batch-invariant across the chunk and item boundaries of the CTA's walk."""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import synth

HERE = os.path.dirname(os.path.abspath(__file__))


def golden_module():
    spec = importlib.util.spec_from_file_location("make_golden_heads", os.path.join(HERE, "golden", "make_golden_heads.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    return mk


MK = golden_module()


@pytest.mark.gpu
@pytest.mark.parametrize("n,h,w,a,c,images", MK.SHAPES, ids=[MK.key(*s[:5]) for s in MK.SHAPES])
def test_matches_the_global_load_heads(golden_dir, n, h, w, a, c, images):
    g = np.load(os.path.join(golden_dir, "heads.npz"))
    got = MK.digests(n, h, w, a, c, images)
    assert len(got) == 10 * len(images)
    for k, v in got.items():
        assert v == str(g[k]), k


def staged(n, h, w, a, c):
    """1 where heads2.a, heads2.b, heads3.a, heads3.b stage their input windows (a record with a window stride), 0 where they read
    the planes, for the plan and workspace a forward of (n, h, w, a, c) runs on."""
    m = MK.make_model(synth.make_state_dict(5, classes=c, anchor_num=a), a, c)
    m(synth.make_images(6, n, h, w).cuda())
    plan = next(iter(m._plans.values()))
    return [int(r["window_stride"] > 0) for r in plan.launches() if r["kernel"].startswith("head")]


@pytest.mark.gpu
def test_window_stride_on_both_sides_of_the_fit_rule():
    """The window (11 rows x 28 floats at 22x22, three 8-channel slots) fits next to the weights of all three kernels with two CTAs
    per SM at 352^2, 640^2 and 150 classes; at 32x2560 the 2x160 map's slot of 6 rows x 164 floats does not, while its 1x80 map
    does; at 4096x32 the 128x1 map's chunks span 128 rows and do not fit either."""
    assert staged(2, 352, 352, 3, 80) == [1, 1, 1, 1]
    assert staged(1, 640, 640, 3, 80) == [1, 1, 1, 1]
    assert staged(2, 96, 128, 3, 150) == [1, 1, 1, 1]
    assert staged(1, 32, 2560, 3, 80) == [0, 0, 1, 1]
    assert staged(1, 4096, 32, 3, 80) == [1, 1, 0, 0]
    import yfv2_engine
    assert yfv2_engine.lib().yfv2_plan_debug_launches(None, None, 0, 0, None, 0, ctypes.byref(ctypes.c_int())) < 0


@pytest.mark.gpu
def test_batch_equals_images_alone():
    """At 256 x 352^2 a CTA walks several (image, 128-pixel chunk) items and stages the next item's first k-steps during the current
    one's last; every image equals, bit for bit, the same image run alone."""
    n = 256
    sd = synth.make_state_dict(91)
    x = synth.make_images(92, n, 352, 352).cuda()
    m = MK.make_model(sd, 3, 80)
    with torch.no_grad():
        big = [p.cpu().numpy() for p in m(x)]
    plan = next(iter(m._plans.values()))
    big_taps = {t: plan.debug_gather(t).cpu().numpy() for t in MK.TAPS}
    m1 = MK.make_model(sd, 3, 80)
    for i in range(n):
        with torch.no_grad():
            one = [p.cpu().numpy() for p in m1(x[i:i + 1])]
        plan1 = next(iter(m1._plans.values()))
        for t in MK.TAPS:
            assert np.array_equal(big_taps[t][i], plan1.debug_gather(t).cpu().numpy()[0]), (t, i)
        for k in range(6):
            assert np.array_equal(big[k][i], one[k][0]), (k, i)

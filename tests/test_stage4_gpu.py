"""Backbone stage 4 on whole images: the stride-2 block stage4.0 runs per image when its 8 warps cover the output map, and
stage4.1-3 run as one chained launch when a whole image fits in one SM's shared memory.  Shapes on both sides of those
selections: 352x352 (both), 224x96 (both), 352x640 (chain only: 11x20 outputs exceed one tile per warp) and 640x640 (neither)."""
import os

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import synth
from oracle import net as onet

pytestmark = pytest.mark.gpu
TOL = dict(rtol=1e-4, atol=1e-4)
SHAPES = [(2, 352, 352), (3, 224, 96), (2, 352, 640), (1, 640, 640)]
TAP = {"stage4.%d" % i: 13 + i for i in range(4)}       # debug_gather index of a block's output
CHAINED = {(352, 352): True, (224, 96): True, (352, 640): True, (640, 640): False}


def make_model(sd):
    import model.detector as det
    m = det.Detector(80, 3, True)
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()


def plan_of(m):
    return next(iter(m._plans.values()))


def run_stage4(plan, x, preds, chained):
    """Runs stage4.0, then stage4.1-3 as one range (one launch where the plan chains them) or one stage at a time; returns the
    taps of every block that is still intact afterwards."""
    names = plan.stage_names
    s40, s43 = names.index("stage4.0"), names.index("stage4.3")
    plan.forward_range(x, preds, s40, s40 + 1)
    taps = {"stage4.0": plan.debug_gather(TAP["stage4.0"]).cpu().numpy()}
    if chained:
        plan.forward_range(x, preds, s40 + 1, s43 + 1)
    else:
        for i in range(s40 + 1, s43 + 1):
            plan.forward_range(x, preds, i, i + 1)
            taps[names[i]] = plan.debug_gather(TAP[names[i]]).cpu().numpy()
    taps["stage4.3"] = plan.debug_gather(TAP["stage4.3"]).cpu().numpy()
    return taps


@pytest.mark.parametrize("n,h,w", SHAPES)
def test_chain_matches_blocks_one_at_a_time(n, h, w):
    sd = synth.make_state_dict(300 + h + w)
    x = synth.make_images(400 + h + w, n, h, w).cuda()
    m = make_model(sd)
    preds = m(x)
    full = [p.clone() for p in preds]
    plan = plan_of(m)
    names, groups = plan.stage_names, plan.stage_groups
    s41 = names.index("stage4.1")
    assert (groups[s41 + 2] == groups[s41]) == CHAINED[(h, w)]
    s40 = names.index("stage4.0")
    plan.forward_range(x, preds, 0, s40)
    chained = run_stage4(plan, x, preds, True)
    plan.forward_range(x, preds, s40 + 4, len(names))
    for p, q in zip(preds, full):
        assert torch.equal(p, q)
    single = run_stage4(plan, x, preds, False)
    for k in ("stage4.0", "stage4.3"):
        assert np.array_equal(chained[k], single[k]), k
    plan.forward_range(x, preds, s40 + 4, len(names))
    for p, q in zip(preds, full):
        assert torch.equal(p, q)


@pytest.mark.parametrize("n,h,w", SHAPES)
def test_stage4_taps_and_heads_against_oracle(n, h, w):
    sd = synth.make_state_dict(500 + h + w)
    xc = synth.make_images(600 + h + w, n, h, w)
    taps = {}
    with torch.no_grad():
        ref = onet.forward(sd, xc, taps=taps)
    x = xc.cuda()
    m = make_model(sd)
    preds = m(x)
    for i, (p, r) in enumerate(zip(preds, ref)):
        np.testing.assert_allclose(p.cpu().numpy(), r.numpy(), err_msg="pred%d" % i, **TOL)
    plan = plan_of(m)
    got = {}
    for chained in (True, False):
        got.update(run_stage4(plan, x, preds, chained))
    assert sorted(got) == sorted(TAP)
    for k, v in got.items():
        np.testing.assert_allclose(v, taps[k].numpy(), err_msg=k, **TOL)


def test_batch_256_equals_batch_1_per_image():
    """Distinct images: a persistent CTA's second image (132 CTAs on an H100) equals the same image run alone."""
    sd = synth.make_state_dict(71)
    x = synth.make_images(72, 256, 352, 352).cuda()
    m = make_model(sd)
    big = [p.clone() for p in m(x)]
    for i in (0, 1, 131, 132, 133, 200, 255):
        one = m(x[i:i + 1])
        for p, q in zip(big, one):
            assert torch.equal(p[i], q[0]), i


@pytest.mark.parametrize("h,w", [(352, 352), (224, 96)])
def test_whole_image_kernels_match_the_banded_kernel(golden_dir, h, w):
    """stage4.0 on the whole-image stride-2 kernel equals, bit for bit, what the banded blk_kernel<96, 2> computed for the same
    image (tests/golden/make_golden_stage4.py), as do the stage4.3 outputs after it."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_golden_stage4", os.path.join(golden_dir, "make_golden_stage4.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    g = np.load(os.path.join(golden_dir, "stage4_banded.npz"))
    got = mk.stage4_taps(h, w)
    for k, v in got.items():
        assert np.array_equal(v, g["%dx%d_%s" % (h, w, k)]), k

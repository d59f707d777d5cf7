"""GPU side of the loss parameter space (tests/loss_space.py) through utils.loss: on every case the device's build_target rows equal
the reference's bit for bit (counts, order, tbox fp32, anch fp64), the four loss scalars are within rtol 1e-5 and d(loss)/d(preds)
within rtol 1e-4 (atol 1e-6 of the largest entry), NaN exactly where the reference has NaN.  The small cases are compared with
the goldens the real reference produced (tests/golden/make_golden_loss_space.py), the large ones with the oracle.  The losses do
not depend on whether gradients are wanted, and two runs give the same bits."""
import os

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import loss_space as ls
import yfv2_engine
from oracle import loss as oloss

pytestmark = pytest.mark.gpu

CASES = {c["name"]: c for c in ls.all_cases()}


@pytest.fixture(scope="module")
def g(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "loss_space.npz")))


def reference(case, g):
    """(build_target arrays, losses[4], grads[6]) of the reference: from the goldens, or the oracle for the large cases."""
    name = case["name"]
    if case["golden"]:
        assert np.array_equal(ls.input_digest(case), g[name + "_digest"])
        bt = {(k, L): g["%s_%s%d" % (name, k, L)] for k in ("tcls", "tbox", "anch", "idx") for L in range(2)}
        return bt, g[name + "_losses"], [g["%s_grad%d" % (name, i)] for i in range(6)]
    preds = [torch.from_numpy(p.copy()).requires_grad_(True) for p in case["preds"]]
    targets = torch.from_numpy(case["targets"].copy())
    tcls, tbox, idx, anch = oloss.build_target(preds, targets, ls.cfg_of(case))
    bt = {}
    for L in range(2):
        bt["tcls", L], bt["tbox", L], bt["anch", L] = tcls[L].numpy(), tbox[L].numpy(), anch[L].numpy()
        bt["idx", L] = torch.stack(idx[L]).numpy()
    out = oloss.compute_loss(preds, targets, ls.cfg_of(case))
    out[3].backward()
    grads = [p.grad.numpy() if p.grad is not None else np.zeros(p.shape, np.float32) for p in preds]
    return bt, np.array([t.item() for t in out]), grads


def bits(t):
    return t.detach().cpu().numpy().view(np.uint32)


@pytest.mark.parametrize("name", list(CASES))
def test_device_loss_equals_reference(g, name):
    import utils.loss as ul
    case = CASES[name]
    bt, ref_losses, ref_grads = reference(case, g)
    cfg = ls.cfg_of(case)
    targets = torch.from_numpy(case["targets"]).cuda()
    preds = [torch.from_numpy(p).cuda().requires_grad_(True) for p in case["preds"]]

    tcls, tbox, indices, anch = ul.build_target(preds, targets, cfg, "cuda")
    for L in range(2):
        assert tbox[L].dtype == torch.float32 and anch[L].dtype == torch.float64
        assert np.array_equal(tcls[L].cpu().numpy(), bt["tcls", L]), L
        assert np.array_equal(tbox[L].cpu().numpy(), bt["tbox", L]), L                 # bit-exact fp32
        assert np.array_equal(anch[L].cpu().numpy(), bt["anch", L]), L                 # bit-exact fp64
        assert np.array_equal(torch.stack(indices[L]).cpu().numpy(), bt["idx", L]), L  # counts and order

    out = ul.compute_loss(preds, targets, cfg, "cuda")
    got = np.array([t.item() for t in out])
    assert np.array_equal(np.isnan(got), np.isnan(ref_losses)), (got, ref_losses)
    np.testing.assert_allclose(got, ref_losses, rtol=1e-5)
    out[3].backward()
    for i, (p, ref) in enumerate(zip(preds, ref_grads)):
        d = p.grad.cpu().numpy()
        assert np.array_equal(np.isnan(d), np.isnan(ref)), "grad%d: NaN in other places than the reference's" % i
        scale = np.abs(ref[np.isfinite(ref)]).max() if np.isfinite(ref).any() else 0.0
        np.testing.assert_allclose(d, ref, rtol=1e-4, atol=1e-6 * max(1e-3, scale), err_msg="grad%d" % i)

    # the losses do not depend on whether gradients are wanted, and a second run gives the same bits (fixed-order reductions)
    dev = [p.detach() for p in preds]
    with_grads, dpreds = yfv2_engine.compute_loss(dev, targets, cfg, want_grads=True)
    without, none = yfv2_engine.compute_loss(dev, targets, cfg, want_grads=False)
    again, dpreds2 = yfv2_engine.compute_loss(dev, targets, cfg, want_grads=True)
    assert none is None
    assert np.array_equal(bits(with_grads), bits(without)) and np.array_equal(bits(with_grads), bits(again))
    assert np.array_equal(bits(with_grads), np.concatenate([bits(t) for t in out]))


def test_mismatched_cfg_is_refused():
    import utils.loss as ul
    case = CASES["borders"]
    preds = [torch.from_numpy(p).cuda() for p in case["preds"]]
    targets = torch.from_numpy(case["targets"]).cuda()
    for key, value in (("anchor_num", 3), ("classes", 80), ("width", 352), ("anchors", case["anchors"] * 2)):
        cfg = ls.cfg_of(case)
        cfg[key] = value
        with pytest.raises(ValueError):
            ul.compute_loss(preds, targets, cfg, "cuda")
    ul.compute_loss(preds, targets, ls.cfg_of(case), "cuda")

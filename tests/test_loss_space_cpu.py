"""CPU side of the loss parameter space (tests/loss_space.py): the oracle against the reference's outputs on every small case, the
numpy restatement of build_target against both, the side every case was built for, the reference's derivative of CIoU at an
exact tie (half of the min / max term to each box), and the cfg / head-shape refusals of yfv2_engine.compute_loss."""
import os

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import loss_space as ls
import yfv2_engine
from oracle import loss as oloss

CASES = {c["name"]: c for c in ls.all_cases()}
GOLDEN = [n for n, c in CASES.items() if c["golden"]]


@pytest.fixture(scope="module")
def g(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "loss_space.npz")))


def oracle_run(case):
    preds = [torch.from_numpy(p.copy()).requires_grad_(True) for p in case["preds"]]
    targets = torch.from_numpy(case["targets"].copy())
    cfg = ls.cfg_of(case)
    bt = oloss.build_target(preds, targets, cfg)
    out = oloss.compute_loss(preds, targets, cfg)
    out[3].backward()
    grads = [p.grad.numpy() if p.grad is not None else np.zeros(p.shape, np.float32) for p in preds]
    return bt, np.array([t.item() for t in out]), grads


def assert_build_target(bt, want, tag):
    """bt: (tcls, tbox, indices, anch) per level as build_target returns them; want(key, L) the expected array."""
    tcls, tbox, indices, anch = bt
    for L in range(2):
        assert np.array_equal(np.asarray(tcls[L]), want("tcls", L)), (tag, L)
        assert np.array_equal(np.asarray(tbox[L]), want("tbox", L)), (tag, L)            # fp32, bit-exact
        assert np.asarray(anch[L]).dtype == np.float64
        assert np.array_equal(np.asarray(anch[L]), want("anch", L)), (tag, L)            # fp64, bit-exact
        assert np.array_equal(np.stack([np.asarray(t) for t in indices[L]], 0), want("idx", L)), (tag, L)


def restated(case):
    out = ([], [], [], [])
    for lv in (0, 1):
        r = ls.rows(case, lv)
        out[0].append(r["cls"]); out[1].append(r["tbox"]); out[2].append((r["b"], r["a"], r["gj"], r["gi"])); out[3].append(r["anch"])
    return out


@pytest.mark.parametrize("name", GOLDEN)
def test_oracle_equals_reference(g, name):
    case = CASES[name]
    assert np.array_equal(ls.input_digest(case), g[name + "_digest"]), "the case builder changed: regenerate the goldens"
    bt, losses, grads = oracle_run(case)
    bt = tuple([[t.numpy() for t in lv] if isinstance(lv, tuple) else lv.numpy() for lv in part] for part in bt)
    assert_build_target(bt, lambda k, L: g["%s_%s%d" % (name, k, L)], name)
    np.testing.assert_allclose(losses, g[name + "_losses"], rtol=1e-6)
    for i in range(6):
        ref = g["%s_grad%d" % (name, i)]
        assert np.array_equal(np.isnan(grads[i]), np.isnan(ref)), (name, i)
        np.testing.assert_allclose(grads[i], ref, rtol=1e-5, atol=1e-9, err_msg="%s grad%d" % (name, i))


@pytest.mark.parametrize("name", list(CASES))
def test_build_target_restatement(g, name):
    """The numpy restatement gives the reference's rows bit for bit (the oracle's for the cases too large to store)."""
    case = CASES[name]
    if case["golden"]:
        want = lambda k, L: g["%s_%s%d" % (name, k, L)]              # noqa: E731
    else:
        preds = [torch.from_numpy(p) for p in case["preds"]]
        tcls, tbox, idx, anch = oloss.build_target(preds, torch.from_numpy(case["targets"]), ls.cfg_of(case))
        ref = {"tcls": tcls, "tbox": tbox, "anch": anch, "idx": [torch.stack(t) for t in idx]}
        want = lambda k, L: ref[k][L].numpy()                         # noqa: E731
    assert_build_target(restated(case), want, name)


@pytest.mark.parametrize("name", list(CASES))
def test_case_sits_on_its_side(name):
    ls.check_sides(CASES[name])


def test_cases_cover_the_space():
    cs = list(CASES.values())
    assert {c["A"] for c in cs} >= {1, 2, 3, 8} and {c["C"] for c in cs} >= {1, 2, 80, 150}
    assert {(c["H"], c["W"]) for c in cs} >= {(32, 32), (64, 96), (512, 512), (352, 640), (640, 640)}
    assert {c["N"] for c in cs} >= {1, 64}
    totals = {5 * c["A"] * len(c["targets"]) for c in cs}
    assert {1020, 1025, 2045, 2050} <= totals                          # 5*A*nt around the 1024-candidate passes
    counts = {c["name"]: [len(ls.rows(c, lv)["b"]) for lv in (0, 1)] for c in cs}
    assert counts["empty"] == [0, 0] and counts["reject_all"] == [0, 0] and counts["reject_level1"][1] == 0
    assert counts["reject_level1"][0] > 0 and len(CASES["reject_all"]["targets"]) > 0
    assert counts["a8_nt3000"][0] > 10000


def test_tie_table():
    """The three tie rows: torch's autograd is the half split of the hand-written reverse mode, the strict comparisons are not."""
    for p, t, tied, want, strict in ls.TIE_TABLE:
        assert ls.box_relation(p, t)["tied"] == tied
        np.testing.assert_allclose(ls.ciou_grad(p, t, 0.5), want, atol=5e-5)
        np.testing.assert_allclose(ls.ciou_grad(p, t, 0.0), strict, atol=5e-5)
        pb = torch.tensor([p], dtype=torch.float64, requires_grad=True)
        oloss.ciou(pb, torch.tensor([t], dtype=torch.float64)).sum().backward()
        np.testing.assert_allclose(pb.grad[0].numpy(), ls.ciou_grad(p, t, 0.5), rtol=1e-12, atol=1e-15)


def test_oracle_gradient_at_ties_is_the_half_split():
    """At every matched row of the CIoU tie case (box logits 0: predicted box (0.5, 0.5, aw, ah)), the oracle's autograd equals
    the reverse mode with half of each tied min / max term, and differs from the strict comparisons exactly where an edge is tied."""
    case = CASES["ciou_ties"]
    n_tied = 0
    for lv in (0, 1):
        r = ls.rows(case, lv)
        for k in range(len(r["b"])):
            p = (0.5, 0.5) + tuple(r["anch"][k])
            t = r["tbox"][k].astype(np.float64)
            rel = ls.box_relation(p, r["tbox"][k])
            assert not rel["identical"]
            pb = torch.tensor([p], dtype=torch.float64, requires_grad=True)
            oloss.ciou(pb, torch.tensor(t[None])).sum().backward()
            half, strict = ls.ciou_grad(p, t, 0.5), ls.ciou_grad(p, t, 0.0)
            np.testing.assert_allclose(pb.grad[0].numpy(), half, rtol=1e-12, atol=1e-15)
            if rel["tied"]:
                n_tied += 1
                assert np.abs(strict - half).max() > 1e-3 * np.abs(half).max(), (lv, k, rel)
            else:
                assert np.array_equal(strict, half)
    assert n_tied >= 4


def test_reference_nan_sits_at_the_zero_size_box(g):
    """The reference's loss is NaN only through lbox, and its gradient is NaN exactly in the four box logits of the cell whose
    predicted box has zero size; a predicted box identical to its target gives no NaN anywhere."""
    losses = g["ciou_nan_losses"]
    assert np.isnan(losses[0]) and np.isfinite(losses[1]) and np.isfinite(losses[2]) and np.isnan(losses[3])
    want = np.zeros(CASES["ciou_nan"]["preds"][0].shape, bool)
    want[0, 0:4, 4, 4] = True
    assert np.array_equal(np.isnan(g["ciou_nan_grad0"]), want)
    assert not any(np.isnan(g["ciou_nan_grad%d" % i]).any() for i in range(1, 6))
    assert np.isfinite(g["ciou_identical_losses"]).all()
    assert all(np.isfinite(g["ciou_identical_grad%d" % i]).all() for i in range(6))


def heads(N, H, W, A, C):
    return [torch.empty(s) for h, w in ls.levels(H, W) for s in ((N, 4 * A, h, w), (N, A, h, w), (N, C, h, w))]


def test_loss_geometry_checks_cfg_against_the_heads():
    cfg = ls.cfg_of(CASES["borders"])                                   # 64x96, A = 2, C = 1
    assert yfv2_engine.loss_geometry(heads(2, 64, 96, 2, 1), cfg) == (2, 64, 96, 2, 1)
    bad = [("anchor_num", 3), ("classes", 80), ("width", 64), ("height", 96), ("width", 352), ("anchors", cfg["anchors"] * 2),
           ("anchors", cfg["anchors"][:4])]
    for key, value in bad:
        c = dict(cfg)
        c[key] = value
        with pytest.raises(ValueError, match=key if key != "width" and key != "height" else "width x height"):
            yfv2_engine.loss_geometry(heads(2, 64, 96, 2, 1), c)
    p = heads(2, 64, 96, 2, 1)
    for i, q in ((3, torch.empty(2, 8, 4, 6)), (4, torch.empty(2, 3, 2, 3)), (5, torch.empty(1, 1, 2, 3)), (2, torch.empty(2, 2, 4, 6))):
        pp = list(p)
        pp[i] = q
        with pytest.raises(ValueError, match="head tensor shapes"):
            yfv2_engine.loss_geometry(pp, cfg)
    with pytest.raises(ValueError, match="six head tensors"):
        yfv2_engine.loss_geometry(p[:3], cfg)

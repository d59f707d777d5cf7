"""GPU: fine-tuning with frozen parameters (requires_grad=False) and BatchNorm modules in .eval() inside a train-mode Detector.

* The eval-mode BatchNorm operators (yfv2_op_bn_eval_fwd / _bwd) against fp64 at the bound of tests/test_train_fp64_gpu.py, over
  ReLU / no ReLU, the float4 / scalar paths and NULL / non-NULL gamma and beta gradients; yfv2_op_bn_train_bwd with NULL gamma /
  beta gradients writes the same dx bit for bit.
* The native trainer under a mode (tests/test_finetune_cpu.py pins which ops and outputs its backward runs): the same head tensors
  and running statistics bit for bit as the unfrozen run when only requires_grad changes, trainable gradients to the fan-out
  order of tests/test_trainer_gpu.py against the unfrozen run and the op-by-op autograd path (model/train_ops.py), with eval-mode
  BatchNorm as close to the fp64 oracle as the reference's own fp32 path; frozen .grad stays None and eval-mode statistics and
  num_batches_tracked stay untouched.
* FlatGradBucket with frozen parameters, mode switches on one model, nothing trainable, and train_dist.py --freeze."""
import gc

import pytest
import torch

import yfv2  # noqa: F401
import synth
from test_finetune_cpu import MASKS, BNNAMES, PNAMES, bn_frozen_stats
from test_train_fp64_gpu import TAU, nerr

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _release_trainers():
    yield
    gc.collect()                  # every Detector owns its trainers' workspaces (several GB at 64x352)
    torch.cuda.empty_cache()


EPS = 1e-5
SHAPES = {"small": (2, 64, 96), "64x352": (64, 352, 352)}
FREEZE_MASKS = ("backbone", "stem+stage2", "stage3", "one-gamma", "shared-obj", "output-only")


# ---- the eval-mode BatchNorm operators ------------------------------------------------------------------------------------
def bn_eval_inputs(seed, N, C, HW):
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g, device="cuda")
    x = r(N, C, HW) * 1.5 + 0.3
    return x, 0.5 + r(C).abs(), 0.2 * r(C), 0.3 * r(C), 0.5 + r(C).abs(), r(N, C, HW)


@pytest.mark.parametrize("affine", ["dgamma+dbeta", "dgamma", "none"])
@pytest.mark.parametrize("HW", [64, 35], ids=["float4", "scalar"])
@pytest.mark.parametrize("relu", [0, 1])
def test_bn_eval_ops_against_fp64(relu, HW, affine):
    import yfv2_engine as eng
    N, C = 3, 5
    x, gamma, beta, rm, rv, dy = bn_eval_inputs(10 + relu + HW, N, C, HW)
    y = torch.empty_like(x)
    mean, invstd = torch.empty(C, device="cuda"), torch.empty(C, device="cuda")
    eng.op("bn_eval_fwd", [x, gamma, beta, rm, rv, y, mean, invstd, N, C, HW, relu], x.device)
    xd, gd, bd = x.double(), gamma.double().view(1, -1, 1), beta.double().view(1, -1, 1)
    mu, inv = rm.double().view(1, -1, 1), (1.0 / torch.sqrt(rv.double() + EPS)).view(1, -1, 1)
    ref = (xd - mu) * inv * gd + bd
    mag = ((xd - mu).abs() + mu.abs()) * inv * gd.abs() + bd.abs()
    if relu:
        ref = ref.clamp_min(0)
    assert torch.equal(mean, rm) and nerr(invstd, inv.view(-1), inv.view(-1)) <= TAU
    assert nerr(y, ref, mag) <= TAU
    dx = torch.empty_like(x)
    dgamma = torch.full((C,), float("nan"), device="cuda") if affine != "none" else None
    dbeta = torch.full((C,), float("nan"), device="cuda") if affine == "dgamma+dbeta" else None
    scratch = torch.empty(2 * C, dtype=torch.float64, device="cuda")
    eng.op("bn_eval_bwd", [x, y, dy, gamma, mean, invstd, dx, dgamma, dbeta, scratch, N, C, HW, relu], x.device)
    d = torch.where(y <= 0, torch.zeros_like(dy), dy).double() if relu else dy.double()
    s = inv * gd
    assert nerr(dx, d * s, d.abs() * s.abs()) <= TAU
    xh = (xd - mean.double().view(1, -1, 1)) * invstd.double().view(1, -1, 1)
    if dgamma is not None:
        assert nerr(dgamma, (d * xh).sum((0, 2)), (d * xh).abs().sum((0, 2))) <= TAU
    if dbeta is not None:
        assert nerr(dbeta, d.sum((0, 2)), d.abs().sum((0, 2))) <= TAU
    # dx may be skipped when only the affine gradients are wanted (a trainable BatchNorm over a frozen input)
    if dgamma is not None:
        g2 = torch.empty_like(dgamma)
        eng.op("bn_eval_bwd", [x, y, dy, gamma, mean, invstd, None, g2, None, scratch, N, C, HW, relu], x.device)
        assert torch.equal(g2, dgamma)


@pytest.mark.parametrize("HW", [64, 35], ids=["float4", "scalar"])
@pytest.mark.parametrize("relu", [0, 1])
def test_bn_train_bwd_without_affine_gradients_keeps_dx(relu, HW):
    import yfv2_engine as eng
    N, C = 3, 5
    x, gamma, beta, _, _, dy = bn_eval_inputs(20 + relu + HW, N, C, HW)
    y = torch.empty_like(x)
    mean, invstd = torch.empty(C, device="cuda"), torch.empty(C, device="cuda")
    scratch = torch.empty(2 * C, dtype=torch.float64, device="cuda")
    eng.op("bn_train_fwd", [x, gamma, beta, None, None, y, mean, invstd, scratch, N, C, HW, relu], x.device)
    dx1, dx2 = torch.empty_like(x), torch.empty_like(x)
    dg, db = torch.empty(C, device="cuda"), torch.empty(C, device="cuda")
    eng.op("bn_train_bwd", [x, y, dy, gamma, mean, invstd, dx1, dg, db, scratch, N, C, HW, relu], x.device)
    eng.op("bn_train_bwd", [x, y, dy, gamma, mean, invstd, dx2, None, None, scratch, N, C, HW, relu], x.device)
    assert torch.equal(dx1, dx2)


# ---- the native trainer under a mode --------------------------------------------------------------------------------------
def make_model(sd, trainable=None, bn_eval=None):
    import model.detector as det
    m = det.Detector(80, 3, True)
    m.load_state_dict(sd, strict=True)
    m = m.cuda().train()
    apply_mode(m, trainable, bn_eval)
    return m


def apply_mode(m, trainable=None, bn_eval=None):
    for p, v in zip(m.parameters(), trainable or [True] * 225):
        p.requires_grad_(bool(v))
    bns = [mod for mod in m.modules() if isinstance(mod, torch.nn.BatchNorm2d)]
    for mod, e in zip(bns, bn_eval or [False] * 73):
        mod.train(not e)


def step(m, x, targets, cfg):
    import utils.loss as ul
    preds = m(x)
    losses = ul.compute_loss(preds, targets, cfg, x.device)
    losses[3].backward()
    bufs = {k: v.clone() for k, v in m.state_dict().items() if "running" in k or "num_batches" in k}
    return ([p.detach().clone() for p in preds], [v.detach().clone() for v in losses],
            [None if p.grad is None else p.grad.detach().clone() for p in m.parameters()], bufs)


_CASES = {}


def case(shape):
    """(state_dict, x, targets, cfg) of a shape"""
    if shape not in _CASES:
        n, h, w = SHAPES[shape]
        _CASES[shape] = (synth.make_state_dict(301), synth.make_images(302, n, h, w).cuda(), synth.make_targets(303, n).cuda(),
                         synth.coco_cfg(w, h))
    return _CASES[shape]


_UNFROZEN = {}


def unfrozen(shape):
    if shape not in _UNFROZEN:
        sd, x, t, cfg = case(shape)
        _UNFROZEN[shape] = step(make_model(sd), x, t, cfg)
    return _UNFROZEN[shape]


def rel(a, b):
    return float((a.double() - b.double()).norm()) / (float(b.double().norm()) + 1e-12)


# Gradients of two runs differ by the order of fan-out sums and fp32 atomics: per tensor 1e-5 relative at the small shape, the
# tolerance of tests/test_trainer_gpu.py.  At 64x352 a stage-2 BatchNorm sums 64*44*44 values per channel and that noise reaches
# 1.6e-5 on backbone tensors, and a beta whose gradient is zero by construction (a BatchNorm without ReLU feeding a 1x1 convolution
# and a train-mode BatchNorm, ~1e-7) is noise only: there the bound is 1e-4 per tensor plus the tensor's share of 1e-4 of the
# global norm, and 1e-4 globally.
TOL = {"small": (1e-5, 0.0, 1e-5), "64x352": (1e-4, 1e-4, 1e-4)}


def assert_grads(got, want, trainable, shape="small"):
    rtol, share, gtol = TOL[shape]
    live = [(i, g, w) for i, (g, w, v) in enumerate(zip(got, want, trainable)) if v]
    assert all(g is None for g, v in zip(got, trainable) if not v), [PNAMES[i] for i, v in enumerate(trainable) if not v and got[i] is not None]
    assert all(g is not None for _, g, _ in live), [PNAMES[i] for i, g, _ in live if g is None]
    total = sum(w.numel() for _, _, w in live)
    wnorm = sum(float(w.double().pow(2).sum()) for _, _, w in live) ** 0.5
    err = sum(float((g.double() - w.double()).pow(2).sum()) for _, g, w in live) ** 0.5
    worst = max((rel(g, w), PNAMES[i]) for i, g, w in live)
    print("gradients: global relative L2 %.2e, worst tensor %.2e (%s)" % (err / wnorm, *worst))
    assert err <= gtol * wnorm
    for i, g, w in live:
        e = float((g.double() - w.double()).norm())
        assert e <= rtol * float(w.double().norm()) + share * wnorm * (w.numel() / total) ** 0.5, (PNAMES[i], rel(g, w))


def run_pyops(monkeypatch, sd, x, t, cfg, trainable, bn_eval):
    from model import train_ops
    with monkeypatch.context() as mp:
        mp.setattr(train_ops, "forward_train_native", train_ops.forward_train)
        return step(make_model(sd, trainable, bn_eval), x, t, cfg)


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("mask", FREEZE_MASKS)
def test_frozen_parameters(mask, shape, monkeypatch):
    sd, x, t, cfg = case(shape)
    trainable = MASKS[mask]
    preds, losses, grads, bufs = step(make_model(sd, trainable), x, t, cfg)
    upreds, ulosses, ugrads, ubufs = unfrozen(shape)
    assert all(torch.equal(a, b) for a, b in zip(preds, upreds))          # the forward does not depend on requires_grad
    assert all(torch.equal(a, b) for a, b in zip(losses, ulosses))
    assert all(torch.equal(bufs[k], ubufs[k]) for k in ubufs)
    assert_grads(grads, ugrads, trainable, shape)                          # only the order of fan-out sums differs
    ppreds, _, pgrads, pbufs = run_pyops(monkeypatch, sd, x, t, cfg, trainable, None)
    assert all(torch.equal(a, b) for a, b in zip(preds, ppreds))
    assert all(torch.equal(bufs[k], pbufs[k]) for k in pbufs)
    assert_grads(grads, pgrads, trainable, shape)


EVAL_MODES = {
    "backbone+freeze-bn": lambda: (MASKS["backbone"], bn_frozen_stats(MASKS["backbone"])),
    "backbone-eval": lambda: (MASKS["all"], [b.startswith("backbone.") for b in BNNAMES]),
    "stem+stage2+freeze-bn": lambda: (MASKS["stem+stage2"], bn_frozen_stats(MASKS["stem+stage2"])),
}


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("mode", list(EVAL_MODES))
def test_eval_mode_batchnorm(mode, shape, monkeypatch):
    sd, x, t, cfg = case(shape)
    trainable, bn_eval = EVAL_MODES[mode]()
    m = make_model(sd, trainable, bn_eval)
    before = {k: v.clone() for k, v in m.state_dict().items() if "running" in k or "num_batches" in k}
    preds, losses, grads, bufs = step(m, x, t, cfg)
    for b, e in zip(BNNAMES, bn_eval):
        for k in ("running_mean", "running_var", "num_batches_tracked"):
            same = torch.equal(bufs[b + "." + k], before[b + "." + k])
            assert same == e or (k != "num_batches_tracked" and not e), (b, k)
    ppreds, plosses, pgrads, pbufs = run_pyops(monkeypatch, sd, x, t, cfg, trainable, bn_eval)
    assert all(torch.equal(a, b) for a, b in zip(preds, ppreds))          # the same kernels in the same order
    assert all(torch.equal(bufs[k], pbufs[k]) for k in pbufs)
    assert_grads(grads, pgrads, trainable, shape)


def _oracle_grads(sd, x, targets, cfg, dtype, trainable, eval_bn):
    import finetune_oracle
    from oracle import loss as oloss
    osd = {k: v.clone().to(dtype) if v.is_floating_point() else v.clone() for k, v in sd.items()}
    for n, v in zip(PNAMES, trainable):
        osd[n].requires_grad_(bool(v))
    preds = finetune_oracle.forward(osd, x.to(dtype), eval_bn)
    oloss.compute_loss(preds, targets, cfg)[3].backward()
    return {n: osd[n].grad.double() for n in PNAMES if osd[n].grad is not None}


@pytest.mark.parametrize("mode", list(EVAL_MODES))
def test_eval_mode_gradients_against_fp64_oracle(mode):
    """The yardstick of tests/test_train_gpu.py: as close to the fp64 oracle as the reference's own fp32 path is."""
    trainable, bn_eval = EVAL_MODES[mode]()
    eval_names = {b for b, e in zip(BNNAMES, bn_eval) if e}
    sd = synth.make_state_dict(61)
    x = synth.make_images(62, 8, 128, 160)
    targets = synth.make_targets(63, 8)
    cfg = synth.coco_cfg(160, 128)
    g32 = _oracle_grads(sd, x, targets, cfg, torch.float32, trainable, eval_names)
    g64 = _oracle_grads(sd, x, targets, cfg, torch.float64, trainable, eval_names)
    _, _, grads, _ = step(make_model(sd, trainable, bn_eval), x.cuda(), targets.cuda(), cfg)
    ours = {n: g.cpu().double() for n, g in zip(PNAMES, grads) if g is not None}
    assert set(ours) == set(g64) == {n for n, v in zip(PNAMES, trainable) if v}

    def relg(a, b):
        return (sum(float((a[k] - b[k]).pow(2).sum()) for k in b) / sum(float(b[k].pow(2).sum()) for k in b)) ** 0.5

    e_ours, e_ref = relg(ours, g64), relg(g32, g64)
    print("%s: global relative L2 vs fp64 oracle: ours %.3e, fp32 oracle %.3e" % (mode, e_ours, e_ref))
    assert e_ours <= max(2.0 * e_ref, 1e-4), (e_ours, e_ref)


# ---- flat bucket, mode switches, nothing trainable ------------------------------------------------------------------------
def test_flat_bucket_with_frozen_parameters():
    import train_ddp
    import utils.loss as ul
    sd = synth.make_state_dict(71)
    x = synth.make_images(72, 2, 96, 96).cuda()
    targets = synth.make_targets(73, 2).cuda()
    cfg = synth.coco_cfg(96, 96)
    trainable = MASKS["backbone"]
    a = make_model(sd, trainable)
    bucket = train_ddp.FlatGradBucket(a.parameters())
    views = [p.grad for p in a.parameters()]
    bucket.zero()
    step(a, x, targets, cfg)
    # the fast path accumulated into the bucket in place: the same .grad objects, no fresh tensors
    assert all(p.grad is v for p, v in zip(a.parameters(), views))
    assert all((p.grad is None) == (not v) for p, v in zip(a.parameters(), trainable))
    offs = a._trainer_for(x).param_offsets
    assert all(p.grad.data_ptr() == bucket.flat.data_ptr() + 4 * off for p, (off, _) in zip(a.parameters(), offs) if off >= 0)
    assert offs[0][0] == -1 and bucket.flat.numel() == a._trainer_for(x).grad_floats
    # three SGD steps through train_ddp.train_step against plain autograd + SGD
    a, b = make_model(sd, trainable), make_model(sd, trainable)
    w0 = [p.detach().clone() for p in a.parameters()]
    bucket = train_ddp.FlatGradBucket(a.parameters())
    opt_a, opt_b = train_ddp.make_optimizer(a, 1e-3), train_ddp.make_optimizer(b, 1e-3)
    for _ in range(3):
        train_ddp.train_step(a, bucket, opt_a, x, targets, cfg, ul.compute_loss)
        ul.compute_loss(b(x), targets, cfg, "cuda")[3].backward()
        opt_b.step()
        opt_b.zero_grad()
    for (n, p1), p2, p0, v in zip(a.named_parameters(), b.parameters(), w0, trainable):
        if not v:
            assert torch.equal(p1, p0) and torch.equal(p2, p0), n
        else:
            torch.testing.assert_close(p1, p2, rtol=1e-5, atol=1e-6, msg=n)


def test_mode_switches_on_one_model():
    """freeze -> unfreeze -> freeze (with eval-mode BatchNorm) on one model: each step equals a fresh model in that mode."""
    sd, x, t, cfg = case("small")
    m = make_model(sd)
    modes = [(MASKS["backbone"], None), (None, None), (MASKS["stem+stage2"], bn_frozen_stats(MASKS["stem+stage2"])),
             (MASKS["backbone"], None)]
    for trainable, bn_eval in modes:
        apply_mode(m, trainable, bn_eval)
        for p in m.parameters():
            p.grad = None
        fresh = make_model({k: v.clone() for k, v in m.state_dict().items()}, trainable, bn_eval)
        got, want = step(m, x, t, cfg), step(fresh, x, t, cfg)
        assert all(torch.equal(a, b) for a, b in zip(got[0], want[0]))
        assert all(torch.equal(got[3][k], want[3][k]) for k in want[3])
        assert_grads(got[2], want[2], trainable or [True] * 225)


def test_nothing_trainable():
    sd, x, t, cfg = case("small")
    import utils.loss as ul
    m = make_model(sd, [False] * 225)
    preds = m(x)
    assert not any(p.requires_grad for p in preds)
    with pytest.raises(RuntimeError):
        ul.compute_loss(preds, t, cfg, x.device)[3].backward()


def test_train_dist_freeze_then_unfreeze(tmp_path, monkeypatch):
    import model.detector as det
    import train_dist
    names = tmp_path / "coco.names"
    names.write_text("\n".join("c%d" % i for i in range(80)) + "\n")
    data = tmp_path / "coco.data"
    data.write_text("[name]\nmodel_name=coco\n\n[train-configure]\nepochs=2\nsteps=150,250\nbatch_size=16\nsubdivisions=1\n"
                    "learning_rate=0.01\n\n[model-configure]\npre_weights=None\nclasses=80\nwidth=352\nheight=352\nanchor_num=3\n"
                    "anchors=12.64,19.39, 37.88,51.48, 55.71,138.31, 126.91,78.23, 131.57,214.55, 279.92,258.87\n\n"
                    "[data-configure]\ntrain=/nonexistent/train.txt\nval=/nonexistent/val.txt\nnames=%s\n" % names)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    monkeypatch.chdir(tmp_path)
    torch.manual_seed(0)                                                  # what train_dist.main builds its model from
    init = {k: v.clone() for k, v in det.Detector(80, 3, True).state_dict().items()}
    args = ["--data", str(data), "--synthetic", "64", "--freeze", "backbone", "--freeze-bn", "--unfreeze-epoch", "1"]
    net0 = train_dist.main(args + ["--epochs", "1"])
    s0 = net0.state_dict()
    assert all(torch.equal(s0[k].cpu(), v) for k, v in init.items() if k.startswith("backbone."))      # weights and BN statistics
    for part in ("bias", "running_mean"):
        assert any(not torch.equal(s0[k].cpu(), v) for k, v in init.items() if k.startswith("fpn.") and k.endswith(part)), part
    assert all(p.grad is None for n, p in net0.named_parameters() if n.startswith("backbone."))
    net1 = train_dist.main(args + ["--epochs", "2"])
    s1 = net1.state_dict()
    for part in ("bias", "running_mean"):
        assert any(not torch.equal(s1[k].cpu(), v) for k, v in init.items() if k.startswith("backbone.") and k.endswith(part)), part
    assert all(p.requires_grad for p in net1.parameters())
    with pytest.raises(SystemExit):
        train_dist.main(["--data", str(data), "--synthetic", "16", "--freeze", "backbone,nonexistent"])

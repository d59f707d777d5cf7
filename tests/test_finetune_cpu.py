"""CPU: fine-tuning with frozen parameters and eval-mode BatchNorm inside a train-mode model.

* The fine-tuning oracle (tests/finetune_oracle.py, autograd over it) against the reference's own Detector fine-tuned on the CPU
  (tests/golden/make_golden_finetune.py): the same parameters receive a gradient, the gradients agree to fp32, and the running
  statistics of eval-mode layers and every num_batches_tracked are bit-identical.
* The native trainer's backward plan for a mode (yfv2_trainer_debug_backward, host only) against the pruning rule restated over
  tests/train_dispatch.py's program: rg(y) = rg(a) | rg(b) | (the op owns a trainable parameter), rg(image) = false; an op runs
  iff rg(y), writes d(a) iff rg(a) and a parameter gradient iff that parameter is trainable.
* The flat layout of a mode against train_ddp.FlatGradBucket's, and the refusals that need no device."""
import ctypes
import os

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import synth
import train_dispatch as td
import finetune_oracle
from oracle import net as onet
from oracle import loss as oloss

SHAPE = (2, 64, 96, 3, 80)


def names():
    """(parameter names in model.parameters() order, BatchNorm module names in module order) of the mirror Detector"""
    import model.detector as det
    m = det.Detector(80, 3, True)
    return ([n for n, _ in m.named_parameters()],
            [n for n, mod in m.named_modules() if isinstance(mod, torch.nn.BatchNorm2d)])


PNAMES, BNNAMES = names()


def freeze(*prefixes):
    return [not n.startswith(prefixes) for n in PNAMES] if prefixes else [True] * len(PNAMES)


def only(*prefixes):
    return [n.startswith(prefixes) for n in PNAMES]


def bn_frozen_stats(trainable):
    """--freeze-bn: eval mode for the layers whose weight and bias are both frozen"""
    tr = dict(zip(PNAMES, trainable))
    return [not tr[b + ".weight"] and not tr[b + ".bias"] for b in BNNAMES]


MASKS = {
    "backbone": freeze("backbone."),
    "stem+stage2": freeze("backbone.first_conv.", "backbone.stage2."),
    "stage3": freeze("backbone.stage3."),                         # d(x) flows through frozen layers into stage2
    "one-gamma": freeze("fpn.conv1x1_2.1.weight"),
    "shared-obj": freeze("output_obj_layers."),
    "output-only": only("output_"),
    "stem-weight-only": freeze("backbone.first_conv.0."),         # a train-mode BatchNorm with trainable affine over a frozen input
    "all": freeze(),
}
BN_MODES = {
    "train": lambda tr: [False] * len(BNNAMES),
    "freeze-bn": bn_frozen_stats,
    "backbone-eval": lambda tr: [b.startswith("backbone.") for b in BNNAMES],
}


# ---- the oracle against the reference ----------------------------------------------------------------------------------------
def load_golden(golden_dir):
    """(the golden's arrays, its generator module: the cases and the sampling of the gradients)"""
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_golden_finetune", os.path.join(golden_dir, "make_golden_finetune.py"))
    mg = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mg)
    return dict(np.load(os.path.join(golden_dir, "finetune_cases.npz"))), mg


@pytest.mark.parametrize("tag", ["frozen_backbone", "backbone_eval", "mixed"])
def test_oracle_matches_the_reference_fine_tuning(golden_dir, tag):
    g, mg = load_golden(golden_dir)
    frozen, eval_prefixes = mg.CASES[tag]
    assert list(g["param_names"]) == PNAMES and list(g[tag + "_bn_names"]) == BNNAMES
    sd = synth.make_state_dict(mg.SEED)
    before = {k: v.clone() for k, v in sd.items()}
    x = synth.make_images(mg.SEED + 1, mg.N, mg.H, mg.W)
    targets = synth.make_targets(mg.SEED + 2, mg.N)
    cfg = synth.coco_cfg(mg.W, mg.H)
    for n in PNAMES:
        sd[n].requires_grad_(not n.startswith(frozen))
    eval_bn = {b for b in BNNAMES if b.startswith(eval_prefixes)}
    assert [b in eval_bn for b in BNNAMES] == list(g[tag + "_bn_eval"])
    preds = finetune_oracle.forward(sd, x, eval_bn, update_running=True)
    losses = oloss.compute_loss(preds, targets, cfg)
    losses[3].backward()
    np.testing.assert_allclose([v.item() for v in losses], g[tag + "_losses"], rtol=1e-5)
    has = [sd[n].grad is not None for n in PNAMES]
    assert has == list(g[tag + "_has_grad"])
    gs = [sd[n].grad.numpy().ravel() for n in PNAMES if sd[n].grad is not None]
    samples = np.concatenate([v[::mg.grad_stride(v.size)] for v in gs])
    norms = np.array([np.linalg.norm(v.astype(np.float64)) for v in gs])
    sums = np.array([v.astype(np.float64).sum() for v in gs])
    # fp32 tolerance of the oracle goldens, scaled to each gradient's size
    scale = np.repeat(g[tag + "_grad_norms"] / np.sqrt([v.size for v in gs]), [v[::mg.grad_stride(v.size)].size for v in gs])
    assert np.all(np.abs(samples - g[tag + "_grad_samples"]) <= 1e-4 * scale + 1e-5 * np.abs(g[tag + "_grad_samples"]))
    np.testing.assert_allclose(norms, g[tag + "_grad_norms"], rtol=1e-4)
    assert np.all(np.abs(sums - g[tag + "_grad_sums"]) <= 1e-4 * g[tag + "_grad_norms"] * np.sqrt([v.size for v in gs]))
    rm = np.concatenate([sd[b + ".running_mean"].numpy() for b in BNNAMES])
    rv = np.concatenate([sd[b + ".running_var"].numpy() for b in BNNAMES])
    nbt = np.array([int(sd[b + ".num_batches_tracked"]) for b in BNNAMES])
    assert np.array_equal(nbt, g[tag + "_nbt"]) and np.array_equal(nbt, [0 if b in eval_bn else 1 for b in BNNAMES])
    off = 0
    for b in BNNAMES:
        c = sd[b + ".running_mean"].numel()
        if b in eval_bn:       # eval mode: untouched, bit for bit, in the oracle and in the reference
            assert np.array_equal(rm[off:off + c], before[b + ".running_mean"].numpy()), b
            assert np.array_equal(g[tag + "_running_mean"][off:off + c], before[b + ".running_mean"].numpy()), b
            assert np.array_equal(g[tag + "_running_var"][off:off + c], before[b + ".running_var"].numpy()), b
        off += c
    # train mode: the existing train-mode oracle tolerance (tests/test_oracle_golden.py)
    np.testing.assert_allclose(rm, g[tag + "_running_mean"], rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(rv, g[tag + "_running_var"], rtol=1e-4, atol=1e-5)


def test_oracle_without_eval_layers_is_the_train_mode_oracle():
    """With no eval-mode layer the fine-tuning oracle is oracle.net's train-mode forward, outputs and buffers bit for bit."""
    sd = synth.make_state_dict(11)
    sd2 = {k: v.clone() for k, v in sd.items()}
    x = synth.make_images(12, 2, 64, 96)
    with torch.no_grad():
        a = onet.forward(sd, x, training=True, update_running=True)
        b = finetune_oracle.forward(sd2, x, (), update_running=True)
        c = finetune_oracle.forward({k: v.clone() for k, v in sd.items()}, x)
    assert all(torch.equal(p, q) for p, q in zip(a, b))
    assert all(torch.equal(sd[k], sd2[k]) for k in sd)
    with torch.no_grad():
        d = onet.forward({k: v.clone() for k, v in sd.items()}, x, training=True)
    assert all(torch.equal(p, q) for p, q in zip(c, d))


# ---- the native trainer's backward plan against the pruning rule -------------------------------------------------------------
def rule(ops, ntens, trainable, bn_eval):
    """The backward plan of the pruning rule, in backward order, as yfv2_trainer_debug_backward reports it."""
    rg = [False] * ntens
    plan = []
    tr = lambda p: p >= 0 and bool(trainable[p])
    for i, o in enumerate(ops):
        dw, dbias, dg, db_ = tr(o["pw"]), tr(o["pbias"]), tr(o["pg"]), tr(o["pb"])
        ra, rb = rg[o["a"]], o["b"] >= 0 and rg[o["b"]]
        run = ra or rb or dw or dbias or dg or db_
        rg[o["y"]] = run
        if run:
            plan.append(dict(op=i, da=int(ra), db=int(rb), dw=int(dw), dbias=int(dbias), dgamma=int(dg), dbeta=int(db_),
                             bn_eval=int(o["kind"] == "bn" and bool(bn_eval[o["bn"]]))))
    return plan[::-1]


def trainer(N, H, W, A, C):
    import yfv2_engine
    lib = yfv2_engine.lib()
    t = ctypes.c_void_p()
    assert lib.yfv2_trainer_create(ctypes.byref(t), 0, N, H, W, A, C) == 0, lib.yfv2_last_error()
    return lib, t


def offsets(lib, t):
    off, num = ctypes.c_longlong(), ctypes.c_longlong()
    out = []
    for i in range(225):
        assert lib.yfv2_trainer_param_offset(t, i, ctypes.byref(off), ctypes.byref(num)) == 0
        out.append((off.value, num.value))
    n = ctypes.c_longlong()
    assert lib.yfv2_trainer_grad_floats(t, ctypes.byref(n)) == 0
    return out, n.value


def test_layer_orders_agree():
    """The trainer's parameter and BatchNorm layer indices are model.parameters() / module order: each BatchNorm op's gamma and
    beta are its layer's weight and bias."""
    ops, _, _ = td.program(*SHAPE)
    for o in ops:
        if o["kind"] == "bn":
            assert PNAMES[o["pg"]] == BNNAMES[o["bn"]] + ".weight" and PNAMES[o["pb"]] == BNNAMES[o["bn"]] + ".bias"


@pytest.mark.parametrize("bn_mode", list(BN_MODES))
@pytest.mark.parametrize("mask", list(MASKS))
def test_backward_plan_follows_the_pruning_rule(mask, bn_mode):
    import yfv2_engine
    import train_ddp
    trainable = MASKS[mask]
    bn_eval = BN_MODES[bn_mode](trainable)
    lib, t = trainer(*SHAPE)
    try:
        yfv2_engine.trainer_set_mode(t, *yfv2_engine.trainer_mode(trainable, bn_eval))
        ops, tens, pnumel = td.program(*SHAPE)
        got = yfv2_engine.trainer_backward_plan(t)
        assert got == rule(ops, len(tens), trainable, bn_eval)
        # written parameter gradients: exactly the trainable parameters
        written = set()
        for r in got:
            o = ops[r["op"]]
            written |= {o[k] for k, f in (("pw", "dw"), ("pbias", "dbias"), ("pg", "dgamma"), ("pb", "dbeta")) if r[f]}
        assert written == {i for i, v in enumerate(trainable) if v}
        # the flat layout is FlatGradBucket's for the same requires_grad flags
        ps = [torch.nn.Parameter(torch.zeros(n), requires_grad=bool(v)) for n, v in zip(pnumel, trainable)]
        bucket = train_ddp.FlatGradBucket(ps)
        offs, total = offsets(lib, t)
        assert total == bucket.flat.numel()
        for p, (off, num), v in zip(ps, offs, trainable):
            assert num == p.numel()
            assert off == (p.grad.data_ptr() - bucket.flat.data_ptr()) // 4 if v else off == -1
    finally:
        lib.yfv2_trainer_destroy(t)


def test_default_mode_runs_every_op_and_writes_every_output():
    import yfv2_engine
    lib, t = trainer(*SHAPE)
    try:
        ops, tens, pnumel = td.program(*SHAPE)
        plan = yfv2_engine.trainer_backward_plan(t)
        assert [r["op"] for r in plan] == list(range(len(ops)))[::-1]
        for r in plan:
            o = ops[r["op"]]
            assert r["da"] == int(tens[o["a"]][3] == -1) and r["db"] == int(o["b"] >= 0)
            assert (r["dw"], r["dbias"], r["dgamma"], r["dbeta"]) == tuple(int(o[k] >= 0) for k in ("pw", "pbias", "pg", "pb"))
            assert r["bn_eval"] == 0
        offs, total = offsets(lib, t)
        assert total == sum(pnumel) and offs == [(sum(pnumel[:i]), n) for i, n in enumerate(pnumel)]
        # setting the default explicitly, or going back to it, gives the same
        yfv2_engine.trainer_set_mode(t, MASKS["backbone"], None)
        yfv2_engine.trainer_set_mode(t, [1] * 225, [0] * 73)
        assert yfv2_engine.trainer_backward_plan(t) == plan and offsets(lib, t) == (offs, total)
    finally:
        lib.yfv2_trainer_destroy(t)


def test_refusals_before_any_launch():
    import yfv2_engine
    lib, t = trainer(*SHAPE)
    fake = ctypes.c_void_p(16)                                       # never dereferenced: the refusals come first
    params = (ctypes.c_void_p * 225)(*[16] * 225)
    heads = (ctypes.c_void_p * 6)(*[16] * 6)

    def backward():
        return lib.yfv2_train_backward(t, fake, params, heads, heads, fake, 0, fake, None)
    try:
        # a mode set after the forward (here: the default mode the trainer was created in) does not apply to its backward
        yfv2_engine.trainer_set_mode(t, MASKS["backbone"], None)
        assert backward() < 0 and b"mode changed after the forward" in lib.yfv2_last_error()
        yfv2_engine.trainer_set_mode(t, [0] * 225, None)
        assert backward() < 0 and b"no parameter is trainable" in lib.yfv2_last_error()
        assert lib.yfv2_trainer_set_mode(t, (ctypes.c_ubyte * 225)(*[2] * 225), None) < 0
        assert b"not 0 or 1" in lib.yfv2_last_error()
        assert lib.yfv2_trainer_set_mode(None, None, None) < 0
    finally:
        lib.yfv2_trainer_destroy(t)
    with pytest.raises(yfv2_engine.Yfv2Error, match="expected 225"):
        yfv2_engine.trainer_mode([True] * 224, None)
    with pytest.raises(yfv2_engine.Yfv2Error, match="expected 73"):
        yfv2_engine.trainer_mode(None, [False] * 74)
    assert yfv2_engine.trainer_mode([True] * 225, [False] * 73) == (None, None)
    # the eval-mode BatchNorm ops: arguments checked before any launch, and no "more than 1 value" refusal
    assert lib.yfv2_op_bn_eval_fwd(*[fake] * 7, None, 1, 8, 1, 1, None) < 0
    assert lib.yfv2_op_bn_eval_bwd(*[fake] * 6, None, None, None, fake, 1, 8, 1, 1, None) < 0    # nothing to write
    assert lib.yfv2_op_bn_eval_bwd(*[fake] * 6, None, fake, None, None, 1, 8, 1, 1, None) < 0    # dgamma without scratch
    assert lib.yfv2_op_bn_train_bwd(*[fake] * 6, None, None, None, fake, 1, 8, 4, 1, None) < 0   # dx stays required


def test_launcher_flags_are_checked():
    import train_dist
    with pytest.raises(SystemExit) as e:
        train_dist.main(["--freeze-bn", "--data", "x.data"])
    assert e.value.code == 2
    with pytest.raises(SystemExit) as e:
        train_dist.main(["--unfreeze-epoch", "1", "--data", "x.data"])
    assert e.value.code == 2

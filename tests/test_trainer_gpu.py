"""The native trainer (csrc/trainer.cu: yfv2_train_forward / yfv2_train_backward, one C-ABI call each) against the op-by-op
autograd composition of the same kernels (model/train_ops.py), which tests/test_train_gpu.py and
tests/test_train_ops_gpu.py pin to the reference: same head tensors and running statistics bit for bit, parameter gradients to
fp32 summation order; gradient accumulation, the flat-bucket fast path and the one-batch-in-flight guard."""
import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import synth

pytestmark = pytest.mark.gpu


def make_model(sd):
    import model.detector as det
    m = det.Detector(80, 3, True)
    m.load_state_dict(sd, strict=True)
    return m.cuda().train()


def run(m, x, targets, cfg):
    import utils.loss as ul
    preds = m(x)
    losses = ul.compute_loss(preds, targets, cfg, x.device)
    losses[3].backward()
    return [p.detach().clone() for p in preds], [l.detach().clone() for l in losses]


def test_native_equals_op_by_op_autograd(monkeypatch):
    sd = synth.make_state_dict(71)
    x = synth.make_images(72, 4, 96, 128).cuda()
    targets = synth.make_targets(73, 4).cuda()
    cfg = synth.coco_cfg(128, 96)
    from model import train_ops
    with monkeypatch.context() as mp:
        mp.setattr(train_ops, "forward_train_native", train_ops.forward_train)
        ma = make_model(sd)
        pa, la = run(ma, x, targets, cfg)
    mb = make_model(sd)
    pb, lb = run(mb, x, targets, cfg)
    for a, b in zip(pa, pb):
        assert torch.equal(a, b)                                     # same kernels in the same order: bit-identical forward
    for a, b in zip(la, lb):
        assert torch.equal(a, b)
    for (k, va), (_, vb) in zip(ma.state_dict().items(), mb.state_dict().items()):
        if "running" in k or "num_batches" in k:
            assert torch.equal(va, vb), k
    for (name, p), (_, q) in zip(ma.named_parameters(), mb.named_parameters()):
        assert p.grad is not None and q.grad is not None, name
        ga, gb = p.grad.double(), q.grad.double()
        denom = float(ga.norm()) + 1e-12
        assert float((ga - gb).norm()) / denom < 1e-5, name             # only the order of fan-out sums differs


def test_flat_bucket_fast_path_and_accumulation():
    import train_ddp
    import utils.loss as ul
    sd = synth.make_state_dict(81)
    x = synth.make_images(82, 2, 64, 96).cuda()
    targets = synth.make_targets(83, 2).cuda()
    cfg = synth.coco_cfg(96, 64)
    m1 = make_model(sd)
    run(m1, x, targets, cfg)                                         # plain autograd: grads returned as views of a fresh flat buffer
    g1 = torch.cat([p.grad.reshape(-1) for p in m1.parameters()])
    m2 = make_model(sd)
    bucket = train_ddp.FlatGradBucket(m2.parameters())               # .grad = consecutive views of one flat buffer: accumulated in place
    bucket.zero()
    run(m2, x, targets, cfg)
    assert all(p.grad.data_ptr() == bucket.flat.data_ptr() + 4 * off for p, (off, _) in zip(m2.parameters(), m2._trainer_for(x).param_offsets))
    # (the weight gradients are reduced with fp32 atomics: run-to-run order noise, compared in relative L2)
    assert float((bucket.flat - g1).double().norm()) / float(g1.double().norm()) < 1e-5
    # a second backward of the same batch accumulates: (the running statistics moved, so compare against a fresh double run)
    m3 = make_model(sd)
    b3 = train_ddp.FlatGradBucket(m3.parameters())
    b3.zero()
    run(m3, x, targets, cfg)
    first = b3.flat.clone()
    run(m3, x, targets, cfg)
    second = b3.flat - first
    # batch-statistics BN: the forward does not depend on the running statistics, so the second gradient equals the first
    assert float((second - first).double().norm()) / float(first.double().norm()) < 1e-5


def test_one_batch_in_flight_guard():
    import utils.loss as ul
    sd = synth.make_state_dict(91)
    x = synth.make_images(92, 2, 64, 64).cuda()
    targets = synth.make_targets(93, 2).cuda()
    cfg = synth.coco_cfg(64, 64)
    m = make_model(sd)
    preds_a = m(x)
    m(x)                                                             # overwrites the workspace of the first forward
    loss = ul.compute_loss(preds_a, targets, cfg, x.device)[3]
    with pytest.raises(RuntimeError, match="ONE batch"):
        loss.backward()

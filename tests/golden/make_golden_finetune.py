"""Generates tests/golden/finetune_cases.npz: the REAL reference Detector (imported from /root/reference) fine-tuned on the CPU, one
training step per case, with parameters frozen (requires_grad=False) and BatchNorm modules put in .eval() inside the train-mode
model, as the usual fine-tuning recipes do.

Run in the build container only (the GPU box has no /root/reference):
    python tests/golden/make_golden_finetune.py [--reference /root/reference]

Per case it stores the four losses of utils/loss.py:compute_loss, which parameters received a .grad (in named_parameters()
order) and those gradients (sampled, with their sums and norms), every BatchNorm layer's running statistics and
num_batches_tracked after the step (the ones before are synth.make_state_dict's).  Inputs come from tests/synth.py, so only
reference outputs are stored; tests/test_finetune_cpu.py pins tests/finetune_oracle.py to them.
"""
import argparse
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

# name -> (frozen parameter-name prefixes, BatchNorm module-name prefixes put in .eval())
CASES = {
    "frozen_backbone": (("backbone.",), ()),
    "backbone_eval": ((), ("backbone.",)),
    # stem + stage2 frozen with their statistics, one FPN gamma frozen, the shared objectness convolution frozen, and one head
    # BatchNorm with frozen statistics but a trainable affine
    "mixed": (("backbone.first_conv.", "backbone.stage2.", "fpn.conv1x1_3.1.weight", "output_obj_layers."),
              ("backbone.first_conv.", "backbone.stage2.", "fpn.cls_head_3.block.1")),
}
SEED, N, H, W = 61, 2, 64, 96


def grad_stride(numel):
    """Every gradient is stored as every k-th element (at most ~256 per parameter), its sum and its L2 norm."""
    return max(1, numel // 256)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default="/root/reference")
    args = ap.parse_args()
    from make_golden import install_shims
    install_shims()
    sys.path.insert(0, args.reference)
    os.chdir(args.reference)
    torch.manual_seed(0)
    import model.detector as rdet
    import utils.loss as rloss
    import synth

    sd = synth.make_state_dict(SEED)
    x = synth.make_images(SEED + 1, N, H, W)
    targets = synth.make_targets(SEED + 2, N)
    cfg = synth.coco_cfg(W, H)
    out = {}
    for tag, (frozen, eval_bn) in CASES.items():
        m = rdet.Detector(80, 3, True)
        m.load_state_dict(sd, strict=True)
        m.train()
        for n, p in m.named_parameters():
            p.requires_grad_(not n.startswith(frozen))
        for n, mod in m.named_modules():
            if isinstance(mod, torch.nn.BatchNorm2d) and n.startswith(eval_bn):
                mod.eval()
        preds = m(x)
        losses = rloss.compute_loss(preds, targets, cfg, torch.device("cpu"))
        losses[3].backward()
        names = [n for n, _ in m.named_parameters()]
        has = np.array([p.grad is not None for _, p in m.named_parameters()])
        out[tag + "_losses"] = np.array([float(v.detach()) for v in losses], np.float32)
        out[tag + "_has_grad"] = has
        gs = [p.grad.detach().numpy().ravel() for _, p in m.named_parameters() if p.grad is not None]
        out[tag + "_grad_samples"] = np.concatenate([g[::grad_stride(g.size)] for g in gs])
        out[tag + "_grad_sums"] = np.array([g.astype(np.float64).sum() for g in gs])
        out[tag + "_grad_norms"] = np.array([np.linalg.norm(g.astype(np.float64)) for g in gs])
        bns = [(n, mod) for n, mod in m.named_modules() if isinstance(mod, torch.nn.BatchNorm2d)]
        out[tag + "_bn_names"] = np.array([n for n, _ in bns])
        out[tag + "_bn_eval"] = np.array([not mod.training for _, mod in bns])
        out[tag + "_running_mean"] = np.concatenate([mod.running_mean.numpy() for _, mod in bns])
        out[tag + "_running_var"] = np.concatenate([mod.running_var.numpy() for _, mod in bns])
        out[tag + "_nbt"] = np.array([int(mod.num_batches_tracked) for _, mod in bns], np.int64)
        out["param_names"] = np.array(names)
    np.savez_compressed(os.path.join(HERE, "finetune_cases.npz"), **out)


if __name__ == "__main__":
    main()

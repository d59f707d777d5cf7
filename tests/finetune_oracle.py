"""CPU oracle of a train-mode Detector.forward with some BatchNorm layers in eval mode (reference model/detector.py:21-47 after
`model.train()` and `.eval()` on those modules, as fine-tuning recipes do).

The same functional restatement as oracle/net.py, whose convolution helpers it uses, with one switch per BatchNorm layer: a layer
named in `eval_bn` normalises with its running statistics and leaves them and num_batches_tracked alone
(F.batch_norm(training=False)); every other layer uses batch statistics and, with `update_running`, updates its running buffers in
`sd` exactly as nn.BatchNorm2d(momentum=0.1, eps=1e-5).train() does.  With an empty `eval_bn` it is
oracle.net.forward(training=True) (tests/test_finetune_cpu.py checks this bit for bit); tests/golden/make_golden_finetune.py pins
it to the reference."""
import torch
import torch.nn.functional as F

from oracle import net as onet


def forward(sd, x, eval_bn=(), update_running=False):
    """(reg_2, obj_2, cls_2, reg_3, obj_3, cls_3) raw logits of the train-mode network; eval_bn: BatchNorm layer names."""
    def bn(t, name):
        w, b = sd[name + ".weight"], sd[name + ".bias"]
        rm, rv = sd[name + ".running_mean"], sd[name + ".running_var"]
        if name in eval_bn:
            return F.batch_norm(t, rm, rv, w, b, False, onet.BN_MOMENTUM, onet.BN_EPS)
        if not update_running:
            return F.batch_norm(t, None, None, w, b, True, onet.BN_MOMENTUM, onet.BN_EPS)
        if (name + ".num_batches_tracked") in sd:
            sd[name + ".num_batches_tracked"] += 1
        return F.batch_norm(t, rm, rv, w, b, True, onet.BN_MOMENTUM, onet.BN_EPS)

    def block(t, pre, stride):                                     # shufflenetv2.py:47-63
        if stride == 1:
            proj, m = t[:, 0::2], t[:, 1::2]
        else:
            proj = bn(onet._dw(sd, t, pre + "branch_proj.0", 2, 1), pre + "branch_proj.1")
            proj = F.relu(bn(onet._pw(sd, proj, pre + "branch_proj.2"), pre + "branch_proj.3"))
            m = t
        m = F.relu(bn(onet._pw(sd, m, pre + "branch_main.0"), pre + "branch_main.1"))
        m = bn(onet._dw(sd, m, pre + "branch_main.3", stride, 1), pre + "branch_main.4")
        m = F.relu(bn(onet._pw(sd, m, pre + "branch_main.5"), pre + "branch_main.6"))
        return torch.cat((proj, m), 1)

    def head(t, pre):                                              # fpn.py:12-29
        for half in (0, 1):
            t = F.relu(bn(onet._dw(sd, t, pre + "block.%d" % (5 * half), 1, 2), pre + "block.%d" % (5 * half + 1)))
            t = bn(onet._pw(sd, t, pre + "block.%d" % (5 * half + 3)), pre + "block.%d" % (5 * half + 4))
        return t

    t = F.conv2d(x, sd["backbone.first_conv.0.weight"], None, 2, 1)    # shufflenetv2.py:74-80,102-109
    t = F.max_pool2d(F.relu(bn(t, "backbone.first_conv.1")), 3, 2, 1)
    outs = []
    for si, rep in enumerate(onet.STAGE_REPEATS):
        for bi in range(rep):
            t = block(t, "backbone.stage%d.%d." % (si + 2, bi), 2 if bi == 0 else 1)
        outs.append(t)
    C2, C3 = outs[1], outs[2]
    S3 = F.relu(bn(onet._pw(sd, C3, "fpn.conv1x1_3.0"), "fpn.conv1x1_3.1"))     # fpn.py:51-64
    cls_3, reg_3 = head(S3, "fpn.cls_head_3."), head(S3, "fpn.reg_head_3.")
    P2 = torch.cat((F.interpolate(C3, scale_factor=2), C2), 1)
    S2 = F.relu(bn(onet._pw(sd, P2, "fpn.conv1x1_2.0"), "fpn.conv1x1_2.1"))
    cls_2, reg_2 = head(S2, "fpn.cls_head_2."), head(S2, "fpn.reg_head_2.")
    return onet.output_layers(sd, cls_2, reg_2) + onet.output_layers(sd, cls_3, reg_3)

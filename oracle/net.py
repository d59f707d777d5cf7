"""Functional CPU restatement of Detector.forward (reference model/detector.py:21-47).

Weights come in as a flat ``state_dict``-style mapping (the reference's 444 keys), so this
file holds no nn.Module tree: each stage is a few torch.nn.functional calls.  With
``training=True`` BatchNorm uses batch statistics (train.py:105 runs the model in
train mode) and, if ``update_running`` is set, the running buffers in ``sd`` are updated
in place exactly as nn.BatchNorm2d(momentum=0.1, eps=1e-5) does.
"""
import torch
import torch.nn.functional as F

BN_EPS = 1e-5       # nn.BatchNorm2d default, used everywhere in the reference
BN_MOMENTUM = 0.1

STAGE_REPEATS = (4, 8, 4)            # model/backbone/shufflenetv2.py:69
STAGE_OUT = (-1, 24, 48, 96, 192)    # model/detector.py:11
FPN_DEPTH = 72                       # model/detector.py:10


def _bn(sd, x, name, training, update_running):
    w, b = sd[name + ".weight"], sd[name + ".bias"]
    rm, rv = sd[name + ".running_mean"], sd[name + ".running_var"]
    if training:
        if update_running:
            y = F.batch_norm(x, rm, rv, w, b, True, BN_MOMENTUM, BN_EPS)
            if (name + ".num_batches_tracked") in sd:
                sd[name + ".num_batches_tracked"] += 1
            return y
        return F.batch_norm(x, None, None, w, b, True, BN_MOMENTUM, BN_EPS)
    return F.batch_norm(x, rm, rv, w, b, False, BN_MOMENTUM, BN_EPS)


def _pw(sd, x, name):
    return F.conv2d(x, sd[name + ".weight"], sd.get(name + ".bias"))


def _dw(sd, x, name, stride, pad):
    w = sd[name + ".weight"]
    return F.conv2d(x, w, None, stride, pad, 1, w.shape[0])


def shuffle_block(sd, x, prefix, stride, training=False, update_running=False):
    """ShuffleV2Block.forward (shufflenetv2.py:47-63)."""
    bn = lambda t, n: _bn(sd, t, prefix + n, training, update_running)
    if stride == 1:
        # channel_shuffle (shufflenetv2.py:57-63): even channels pass, odd go to main
        proj, m = x[:, 0::2], x[:, 1::2]
    else:
        # branch_proj: dw s2 + BN -> pw + BN + ReLU (shufflenetv2.py:34-44)
        proj = bn(_dw(sd, x, prefix + "branch_proj.0", 2, 1), "branch_proj.1")
        proj = F.relu(bn(_pw(sd, proj, prefix + "branch_proj.2"), "branch_proj.3"))
        m = x
    # branch_main: pw+BN+ReLU -> dw+BN -> pw+BN+ReLU (shufflenetv2.py:19-32)
    m = F.relu(bn(_pw(sd, m, prefix + "branch_main.0"), "branch_main.1"))
    m = bn(_dw(sd, m, prefix + "branch_main.3", stride, 1), "branch_main.4")
    m = F.relu(bn(_pw(sd, m, prefix + "branch_main.5"), "branch_main.6"))
    return torch.cat((proj, m), 1)


def stem(sd, x, training=False, update_running=False):
    """first_conv + maxpool (shufflenetv2.py:74-80,103-104)."""
    p = "backbone."
    x = F.conv2d(x, sd[p + "first_conv.0.weight"], None, 2, 1)
    x = F.relu(_bn(sd, x, p + "first_conv.1", training, update_running))
    return F.max_pool2d(x, 3, 2, 1)


def backbone(sd, x, training=False, update_running=False, taps=None):
    """ShuffleNetV2.forward (shufflenetv2.py:102-109) -> (C2, C3)."""
    p = "backbone."
    x = stem(sd, x, training, update_running)
    if taps is not None:
        taps["stem"] = x
    outs = []
    for si, rep in enumerate(STAGE_REPEATS):
        for bi in range(rep):
            pre = "%sstage%d.%d." % (p, si + 2, bi)
            x = shuffle_block(sd, x, pre, 2 if bi == 0 else 1, training, update_running)
            if taps is not None:
                taps["stage%d.%d" % (si + 2, bi)] = x
        outs.append(x)
    return outs[1], outs[2]


def dwconv_half(sd, x, prefix, half, training=False, update_running=False):
    """One half of DWConvblock.forward (fpn.py:12-29): dw5x5+BN+ReLU, pw+BN; half 0 is block.0-4, half 1 block.5-9."""
    bn = lambda t, i: _bn(sd, t, prefix + "block.%d" % (i + 5 * half), training, update_running)
    x = F.relu(bn(_dw(sd, x, prefix + "block.%d" % (5 * half), 1, 2), 1))
    return bn(_pw(sd, x, prefix + "block.%d" % (3 + 5 * half)), 4)


def dwconv_block(sd, x, prefix, training=False, update_running=False):
    """DWConvblock.forward (fpn.py:12-29): dw5x5+BN+ReLU, pw+BN, dw5x5+BN+ReLU, pw+BN."""
    x = dwconv_half(sd, x, prefix, 0, training, update_running)
    return dwconv_half(sd, x, prefix, 1, training, update_running)


def reduce_s3(sd, C3, training=False, update_running=False):
    """S3 = conv1x1_3(C3) + BN + ReLU (fpn.py:51-52)."""
    p = "fpn.conv1x1_3."
    return F.relu(_bn(sd, _pw(sd, C3, p + "0"), p + "1", training, update_running))


def reduce_s2(sd, C2, C3, training=False, update_running=False):
    """S2 = conv1x1_2(cat(nearest-up2(C3), C2)) + BN + ReLU (fpn.py:57-59)."""
    p = "fpn.conv1x1_2."
    P2 = torch.cat((F.interpolate(C3, scale_factor=2), C2), 1)
    return F.relu(_bn(sd, _pw(sd, P2, p + "0"), p + "1", training, update_running))


def fpn(sd, C2, C3, training=False, update_running=False, taps=None):
    """LightFPN.forward (fpn.py:51-64).  Module execution order matters in train mode only
    through running-stat updates, which are per-layer, so order is free here."""
    p = "fpn."
    S3 = reduce_s3(sd, C3, training, update_running)
    cls_3 = dwconv_block(sd, S3, p + "cls_head_3.", training, update_running)
    reg_3 = dwconv_block(sd, S3, p + "reg_head_3.", training, update_running)
    S2 = reduce_s2(sd, C2, C3, training, update_running)
    cls_2 = dwconv_block(sd, S2, p + "cls_head_2.", training, update_running)
    reg_2 = dwconv_block(sd, S2, p + "reg_head_2.", training, update_running)
    if taps is not None:
        taps.update(S2=S2, S3=S3, cls_2=cls_2, reg_2=reg_2, cls_3=cls_3, reg_3=reg_3)
    return cls_2, reg_2, cls_3, reg_3


def forward(sd, x, training=False, update_running=False, taps=None):
    """Detector.forward, export_onnx=False branch (detector.py:21-31,46-47).

    Returns (reg_2, obj_2, cls_2, reg_3, obj_3, cls_3) raw logits, NCHW fp32."""
    C2, C3 = backbone(sd, x, training, update_running, taps)
    if taps is not None:
        taps["C2"], taps["C3"] = C2, C3
    cls_2, reg_2, cls_3, reg_3 = fpn(sd, C2, C3, training, update_running, taps)
    return output_layers(sd, cls_2, reg_2) + output_layers(sd, cls_3, reg_3)


def output_layers(sd, cls_f, reg_f):
    """(reg, obj, cls) logits of one level (detector.py:17-19,28-31)."""
    return (_pw(sd, reg_f, "output_reg_layers"),
            _pw(sd, cls_f, "output_obj_layers"),      # obj aliases the cls branch, fpn.py:54,61
            _pw(sd, cls_f, "output_cls_layers"))


def forward_export(sd, x):
    """export_onnx=True branch (detector.py:33-44): two NHWC [N,h,w,4A+A+C] tensors."""
    o = forward(sd, x)
    res = []
    for i in (0, 3):
        t = torch.cat((o[i].sigmoid(), o[i + 1].sigmoid(), F.softmax(o[i + 2], dim=1)), 1)
        res.append(t.permute(0, 2, 3, 1))
    return tuple(res)

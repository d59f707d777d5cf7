"""Train-mode network (SURVEY 8 row a13): batch-statistics BatchNorm forward and the backward of every op, as
torch.autograd.Function wrappers around the C-ABI training operators of libyfv2.so (csrc/k_train.cu).  Autograd only keeps
the graph; all arithmetic (1x1 / depthwise / stem convolutions and their dgrad / wgrad, BatchNorm statistics and its
backward, ReLU masks, max-pool, up-sampling) runs in our kernels.  Channel shuffle / split / concat are index plumbing and
use torch indexing.  Mirrors the reference's train-mode Detector.forward (model/detector.py:21-31 with nn.Module.train())."""
import torch
import torch.nn as nn

import yfv2_engine as eng


def _c(t):
    return t if t.is_contiguous() else t.contiguous()


class Conv1x1(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, bias):
        x = _c(x)
        N, K, H, W = x.shape
        M = w.shape[0]
        y = torch.empty((N, M, H, W), dtype=torch.float32, device=x.device)
        eng.op("conv1x1_fwd", [x, w, bias, y, N, K, M, H * W], x.device)
        ctx.save_for_backward(x, w)
        ctx.has_bias = bias is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        dy = _c(dy)
        N, K, H, W = x.shape
        M = w.shape[0]
        dx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        dw = torch.empty_like(w) if ctx.needs_input_grad[1] else None
        db = torch.empty(M, dtype=torch.float32, device=x.device) if ctx.has_bias and ctx.needs_input_grad[2] else None
        eng.op("conv1x1_bwd", [x, w, dy, dx, dw, db, N, K, M, H * W], x.device)
        return dx, dw, db


class DwConv(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, stride):
        x = _c(x)
        N, C, H, W = x.shape
        ks = w.shape[-1]
        Ho, Wo = (H + 2 * (ks // 2) - ks) // stride + 1, (W + 2 * (ks // 2) - ks) // stride + 1
        y = torch.empty((N, C, Ho, Wo), dtype=torch.float32, device=x.device)
        eng.op("dwconv_fwd", [x, w, y, N, C, H, W, ks, stride], x.device)
        ctx.save_for_backward(x, w)
        ctx.stride = stride
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        dy = _c(dy)
        N, C, H, W = x.shape
        ks = w.shape[-1]
        dx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        dw = torch.empty_like(w) if ctx.needs_input_grad[1] else None
        eng.op("dwconv_bwd", [x, w, dy, dx, dw, N, C, H, W, ks, ctx.stride], x.device)
        return dx, dw, None


class StemConv(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w):
        x = _c(x)
        N, _, H, W = x.shape
        M = w.shape[0]
        y = torch.empty((N, M, H // 2, W // 2), dtype=torch.float32, device=x.device)
        eng.op("stem_fwd", [x, w, y, N, M, H, W], x.device)
        ctx.save_for_backward(x, w)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        if ctx.needs_input_grad[0]:
            raise NotImplementedError("gradient with respect to the input image is not implemented (train.py never asks for it)")
        N, _, H, W = x.shape
        dw = torch.empty_like(w)
        eng.op("stem_wgrad", [x, _c(dy), dw, N, w.shape[0], H, W], x.device)
        return None, dw


class BnTrain(torch.autograd.Function):
    """y = [ReLU](BN_train(x)); updates running_mean / running_var in place like nn.BatchNorm2d.train()."""

    @staticmethod
    def forward(ctx, x, gamma, beta, running_mean, running_var, relu):
        x = _c(x)
        N, C, H, W = x.shape
        if N * H * W == 1:                                   # F.batch_norm's refusal (the kernel refuses it too)
            raise ValueError("Expected more than 1 value per channel when training, got input size %s" % (x.shape,))
        y = torch.empty_like(x)
        mean = torch.empty(C, dtype=torch.float32, device=x.device)
        invstd = torch.empty(C, dtype=torch.float32, device=x.device)
        scratch = torch.empty(2 * C, dtype=torch.float64, device=x.device)
        eng.op("bn_train_fwd", [x, gamma, beta, running_mean, running_var, y, mean, invstd, scratch, N, C, H * W, int(relu)], x.device)
        ctx.save_for_backward(x, y, gamma, mean, invstd)
        ctx.relu = int(relu)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, y, gamma, mean, invstd = ctx.saved_tensors
        N, C, H, W = x.shape
        dx = torch.empty_like(x)                             # (needed for the sums even when x needs no gradient)
        dgamma = torch.empty_like(gamma) if ctx.needs_input_grad[1] else None
        dbeta = torch.empty_like(gamma) if ctx.needs_input_grad[2] else None
        scratch = torch.empty(2 * C, dtype=torch.float64, device=x.device)
        eng.op("bn_train_bwd", [x, y, _c(dy), gamma, mean, invstd, dx, dgamma, dbeta, scratch, N, C, H * W, ctx.relu], x.device)
        return (dx if ctx.needs_input_grad[0] else None), dgamma, dbeta, None, None, None


class BnEval(torch.autograd.Function):
    """y = [ReLU](BN_eval(x)): a BatchNorm module in .eval() inside a train-mode network (running statistics, not updated)."""

    @staticmethod
    def forward(ctx, x, gamma, beta, running_mean, running_var, relu):
        x = _c(x)
        N, C, H, W = x.shape
        y = torch.empty_like(x)
        mean = torch.empty(C, dtype=torch.float32, device=x.device)
        invstd = torch.empty(C, dtype=torch.float32, device=x.device)
        eng.op("bn_eval_fwd", [x, gamma, beta, running_mean, running_var, y, mean, invstd, N, C, H * W, int(relu)], x.device)
        ctx.save_for_backward(x, y, gamma, mean, invstd)
        ctx.relu = int(relu)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, y, gamma, mean, invstd = ctx.saved_tensors
        N, C, H, W = x.shape
        dx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        dgamma = torch.empty_like(gamma) if ctx.needs_input_grad[1] else None
        dbeta = torch.empty_like(gamma) if ctx.needs_input_grad[2] else None
        scratch = torch.empty(2 * C, dtype=torch.float64, device=x.device) if dgamma is not None or dbeta is not None else None
        eng.op("bn_eval_bwd", [x, y, _c(dy), gamma, mean, invstd, dx, dgamma, dbeta, scratch, N, C, H * W, ctx.relu], x.device)
        return dx, dgamma, dbeta, None, None, None


class MaxPool3x3s2(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        x = _c(x)
        N, C, H, W = x.shape
        Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        y = torch.empty((N, C, Ho, Wo), dtype=torch.float32, device=x.device)
        idx = torch.empty((N, C, Ho, Wo), dtype=torch.int32, device=x.device)
        eng.op("maxpool_fwd", [x, y, idx, N * C, H, W], x.device)
        ctx.save_for_backward(idx)
        ctx.shape = (N, C, H, W)
        return y

    @staticmethod
    def backward(ctx, dy):
        (idx,) = ctx.saved_tensors
        N, C, H, W = ctx.shape
        dx = torch.empty((N, C, H, W), dtype=torch.float32, device=dy.device)
        eng.op("maxpool_bwd", [_c(dy), idx, dx, N * C, H, W], dy.device)
        return dx


class Upsample2x(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        x = _c(x)
        N, C, H, W = x.shape
        y = torch.empty((N, C, 2 * H, 2 * W), dtype=torch.float32, device=x.device)
        eng.op("upsample2_fwd", [x, y, N * C, H, W], x.device)
        ctx.shape = (N, C, H, W)
        return y

    @staticmethod
    def backward(ctx, dy):
        N, C, H, W = ctx.shape
        dx = torch.empty((N, C, H, W), dtype=torch.float32, device=dy.device)
        eng.op("upsample2_bwd", [_c(dy), dx, N * C, H, W], dy.device)
        return dx


# ---- network composition (same wiring as the eval engine, module parameters as weights) ---------------------------------
def _bn(x, bn, relu):
    if not bn.training:                                      # e.g. model.backbone.eval() inside a train-mode model
        return BnEval.apply(x, bn.weight, bn.bias, bn.running_mean, bn.running_var, relu)
    y = BnTrain.apply(x, bn.weight, bn.bias, bn.running_mean, bn.running_var, relu)
    bn.num_batches_tracked += 1
    return y


def _pw_bn(x, conv, bn, relu):
    return _bn(Conv1x1.apply(x, conv.weight, None), bn, relu)


def _dw_bn(x, conv, bn, relu):
    return _bn(DwConv.apply(x, conv.weight, conv.stride[0]), bn, relu)


def _shuffle_block(blk, x):
    m = blk.branch_main
    if blk.stride == 1:
        proj, xm = x[:, 0::2], x[:, 1::2]                       # channel_shuffle: even pass, odd -> main (shufflenetv2.py:57-63)
    else:
        p = blk.branch_proj
        proj = _pw_bn(_dw_bn(x, p[0], p[1], False), p[2], p[3], True)
        xm = x
    xm = _pw_bn(xm, m[0], m[1], True)
    xm = _dw_bn(xm, m[3], m[4], False)
    xm = _pw_bn(xm, m[5], m[6], True)
    return torch.cat((proj, xm), 1)


def _head(block, x):
    b = block.block
    x = _dw_bn(x, b[0], b[1], True)
    x = _pw_bn(x, b[3], b[4], False)
    x = _dw_bn(x, b[5], b[6], True)
    return _pw_bn(x, b[8], b[9], False)


# ---- the whole network as ONE autograd node over the native trainer (csrc/trainer.cu) ------------------------------------------
class NetTrainFn(torch.autograd.Function):
    """preds = net(x) in train mode.  forward: yfv2_train_forward (saves activations in the trainer's workspace); backward:
    yfv2_train_backward -> every trainable parameter's gradient in one flat buffer.  When the trainable parameters' .grad already
    are the consecutive views of one flat buffer in parameter order (train_ddp.FlatGradBucket), the gradients are ACCUMULATED
    straight into it and autograd is told there is nothing more to add; otherwise they are returned as views of a fresh flat
    buffer.  Frozen parameters (requires_grad=False) get None, and BatchNorm modules in .eval() run on their running statistics:
    the trainer's mode follows both on every call."""

    @staticmethod
    def forward(ctx, x, model, *params):
        if x.requires_grad:
            raise NotImplementedError("gradient with respect to the input image is not implemented (train.py never asks for it)")
        tr = model._trainer_for(x)
        bn, nbt = model._train_buffers()
        bn_eval = [not m.training for m in model._bn_modules()]
        tr.set_mode([p.requires_grad for p in params], bn_eval)
        plist = [p.detach() for p in params]
        preds = tr.forward(x, plist, bn)
        if any(bn_eval):                                 # an eval-mode layer does not count the batch (nn.BatchNorm2d.forward)
            nbt = [t for t, e in zip(nbt, bn_eval) if not e]
        if nbt:
            torch._foreach_add_(nbt, 1)
        ctx.tr, ctx.gen, ctx.plist, ctx.params = tr, tr.generation, plist, params
        return tuple(preds)

    @staticmethod
    def backward(ctx, *dpreds):
        tr = ctx.tr
        if tr.generation != ctx.gen:
            raise RuntimeError("yfv2: the native trainer keeps ONE batch's activations per input shape; call backward() before the next "
                               "train-mode forward of that shape")
        # the trainable parameters, each with its slot of the flat buffer (frozen ones have offset -1)
        live = [(p, off, num) for p, (off, num) in zip(ctx.params, tr.param_offsets) if off >= 0]
        # fast path: .grad tensors are the slices of one flat bucket, in order
        base = None
        if live and all(p.grad is not None and p.grad.is_contiguous() and p.grad.dtype == torch.float32 for p, _, _ in live):
            base = live[0][0].grad.data_ptr()
            for p, off, num in live:
                if p.grad.data_ptr() != base + 4 * off or p.grad.numel() != num:
                    base = None
                    break
        if base is not None:
            g0 = live[0][0].grad
            flat = torch.as_strided(g0, (tr.grad_floats,), (1,), g0.storage_offset()) if g0.untyped_storage().nbytes() >= 4 * (g0.storage_offset() + tr.grad_floats) else None
            if flat is not None:
                tr.backward(ctx.plist, dpreds, flat, accumulate=True)
                return (None, None) + tuple(None for _ in ctx.params)
        flat = tr.backward(ctx.plist, dpreds, None, accumulate=False).clone()      # (autograd may keep what it is handed as .grad)
        return (None, None) + tuple(flat[off:off + num].view_as(p) if off >= 0 else None for p, (off, num) in zip(ctx.params, tr.param_offsets))


def forward_train_native(model, x):
    """Train-mode Detector.forward through the native trainer: one autograd node for the whole network."""
    return NetTrainFn.apply(x.contiguous(), model, *model.parameters())


def forward_train(model, x):
    """Train-mode Detector.forward: returns the six raw head tensors with an autograd graph over our kernels."""
    bb, fpn = model.backbone, model.fpn
    x = _bn(StemConv.apply(x, bb.first_conv[0].weight), bb.first_conv[1], True)
    x = MaxPool3x3s2.apply(x)
    feats = []
    for name in ("stage2", "stage3", "stage4"):
        for blk in getattr(bb, name):
            x = _shuffle_block(blk, x)
        feats.append(x)
    C2, C3 = feats[1], feats[2]
    S3 = _pw_bn(C3, fpn.conv1x1_3[0], fpn.conv1x1_3[1], True)
    cls_3, reg_3 = _head(fpn.cls_head_3, S3), _head(fpn.reg_head_3, S3)
    P2 = torch.cat((Upsample2x.apply(C3), C2), 1)
    S2 = _pw_bn(P2, fpn.conv1x1_2[0], fpn.conv1x1_2[1], True)
    cls_2, reg_2 = _head(fpn.cls_head_2, S2), _head(fpn.reg_head_2, S2)
    out = []
    for cls_f, reg_f in ((cls_2, reg_2), (cls_3, reg_3)):
        out.append(Conv1x1.apply(reg_f, model.output_reg_layers.weight, model.output_reg_layers.bias))
        out.append(Conv1x1.apply(cls_f, model.output_obj_layers.weight, model.output_obj_layers.bias))
        out.append(Conv1x1.apply(cls_f, model.output_cls_layers.weight, model.output_cls_layers.bias))
    return tuple(out)

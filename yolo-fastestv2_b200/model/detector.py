"""Drop-in replacement for the reference's model/detector.py:Detector.

Same constructor and forward signature, same sub-module tree (hence the same 444 state_dict keys, so
modelzoo checkpoints load with strict=True), but forward() runs the fused CUDA kernels of libyfv2.so
through the C ABI (include/yfv2.h).  CUDA only: a CPU tensor raises — there is no fallback path.
"""
import os
import sys

import torch
import torch.nn as nn

_PKG = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if _PKG not in sys.path:
    sys.path.insert(0, _PKG)

import yfv2_engine                                           # noqa: E402
from model.fpn import LightFPN                               # noqa: E402
from model.backbone.shufflenetv2 import ShuffleNetV2         # noqa: E402


class Detector(nn.Module):
    def __init__(self, classes, anchor_num, load_param, export_onnx=False):
        super().__init__()
        out_depth = 72
        stage_out_channels = [-1, 24, 48, 96, 192]
        self.export_onnx = export_onnx
        self.classes, self.anchor_num = classes, anchor_num
        self.backbone = ShuffleNetV2(stage_out_channels, load_param)
        self.fpn = LightFPN(stage_out_channels[-2] + stage_out_channels[-1], stage_out_channels[-1], out_depth)
        self.output_reg_layers = nn.Conv2d(out_depth, 4 * anchor_num, 1, 1, 0, bias=True)
        self.output_obj_layers = nn.Conv2d(out_depth, anchor_num, 1, 1, 0, bias=True)
        self.output_cls_layers = nn.Conv2d(out_depth, classes, 1, 1, 0, bias=True)
        self._plans = {}
        self._trainers = {}
        self._weights_gen = 0           # bumped whenever weights / BN buffers may have changed behind autograd's back

    # ---- weight bookkeeping ---------------------------------------------------------------------------
    def _weight_tensors(self):
        params = list(self.parameters())
        bn = []
        for m in self.modules():
            if isinstance(m, nn.BatchNorm2d):
                bn += [m.running_mean, m.running_var]
        return params, bn

    def _train_buffers(self):
        """(running_mean / running_var list, num_batches_tracked list) for the native trainer; the module walk is cached and
        re-done when `.to()` / `.cuda()` / load_state_dict replaced the buffer tensors."""
        c = self.__dict__.get("_train_buf_cache")
        first = self.backbone.first_conv[1]
        if c is None or c[2] is not first.running_mean or c[3] is not first.num_batches_tracked:
            bn, nbt = [], []
            for m in self.modules():
                if isinstance(m, nn.BatchNorm2d):
                    bn += [m.running_mean, m.running_var]
                    nbt.append(m.num_batches_tracked)
            c = (bn, nbt, first.running_mean, first.num_batches_tracked)
            self.__dict__["_train_buf_cache"] = c
        return c[0], c[1]

    def invalidate_packed(self):
        """Forces the next eval forward to re-fold BN and re-pack the weights.  Needed after edits that do not bump
        `tensor._version` (`p.data.add_()`, raw-pointer updates); `forward()` in train mode and `load_state_dict` call it."""
        self._weights_gen += 1

    def load_state_dict(self, *a, **k):
        r = super().load_state_dict(*a, **k)
        self.invalidate_packed()
        return r

    # plans hold ctypes handles and device buffers: copies / pickles of the module start without them and re-pack lazily
    def __deepcopy__(self, memo):
        import copy
        cls = self.__class__
        new = cls.__new__(cls)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            if k == "_train_buf_cache":
                continue
            new.__dict__[k] = {} if k in ("_plans", "_trainers") else copy.deepcopy(v, memo)
        return new

    def __getstate__(self):
        st = dict(self.__dict__)
        st["_plans"] = {}
        st["_trainers"] = {}
        st.pop("_train_buf_cache", None)
        return st

    def _trainer_for(self, x):
        N, _, H, W = x.shape
        key = (x.device.index, N, H, W)
        tr = self._trainers.get(key)
        if tr is None:
            if len(self._trainers) >= 4:
                self._trainers.pop(next(iter(self._trainers)))
            tr = yfv2_engine.Trainer(x.device, N, H, W, self.anchor_num, self.classes)
            self._trainers[key] = tr
        return tr

    def _plan_for(self, x):
        N, _, H, W = x.shape
        key = (x.device.index, N, H, W)
        plan = self._plans.get(key)
        if plan is None:
            if len(self._plans) >= 8:
                self._plans.pop(next(iter(self._plans)))
            plan = yfv2_engine.Plan(x.device, N, H, W, self.anchor_num, self.classes, training=False)
            self._plans[key] = plan
        params, bn = self._weight_tensors()
        version = (self._weights_gen,) + tuple(t._version for t in params + bn) + tuple(t.data_ptr() for t in params[:1])
        if plan.packed_version != version:
            plan.pack(params, bn)
            plan.packed_version = version
        return plan

    # ---- forward -----------------------------------------------------------------------------------------
    def forward(self, x):
        if not x.is_cuda:
            raise RuntimeError("yfv2 Detector runs on CUDA only (no CPU fallback); move the model and input to a GPU")
        if self.training:
            if self.export_onnx:
                raise NotImplementedError("export_onnx=True is an inference-only head")
            from model import train_ops
            self.invalidate_packed()                      # the BN running statistics are updated through raw pointers
            x = x.float() if x.dtype != torch.float32 else x
            yfv2_engine.check_bn_batch(x.shape[0], x.shape[2], x.shape[3])
            # default: the native trainer (csrc/trainer.cu), one C-ABI call for the forward and one for the backward;
            # YFV2_TRAIN_PYOPS=1 keeps the op-by-op autograd composition (the path the operator tests pin)
            if os.environ.get("YFV2_TRAIN_PYOPS") or x.shape[2] % 32 or x.shape[3] % 32:
                return train_ops.forward_train(self, x)
            return train_ops.forward_train_native(self, x)
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError("expected input [N,3,H,W]")
        plan = self._plan_for(x)
        if x.dtype not in (torch.float32, torch.uint8):
            x = x.float()
        preds = plan.forward(x)
        if self.export_onnx:
            print("export onnx ...")                      # the reference prints this on every export-mode forward
            return yfv2_engine.export_heads(preds)
        return preds

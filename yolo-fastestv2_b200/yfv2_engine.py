"""ctypes binding of libyfv2.so (include/yfv2.h) plus the small amount of host bookkeeping the Python
mirror modules share: plan cache, weight packing, output allocation.  PyTorch is used for device
memory and streams only; every device computation is a kernel inside libyfv2.so.

There is NO CPU fallback: if the library is missing or the tensors are not on a CUDA device the calls
raise.
"""
import ctypes
import os
import threading

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libyfv2.so")
_lib = None
_lock = threading.Lock()

MAX_DET = 300          # reference utils/utils.py:242
MAX_WH = 4096.0        # reference utils/utils.py:241

_c_float_p = ctypes.POINTER(ctypes.c_float)
_c_void_pp = ctypes.POINTER(ctypes.c_void_p)


class Frame(ctypes.Structure):
    """yfv2_frame: one packed HWC BGR uint8 source frame in device memory."""
    _fields_ = [("data", ctypes.c_void_p), ("w", ctypes.c_int), ("h", ctypes.c_int), ("pitch", ctypes.c_longlong)]


class Yuv420Frame(ctypes.Structure):
    """yfv2_yuv420_frame: one YUV 4:2:0 source frame (NV12 / NV21 / I420 / YV12) in device memory."""
    _fields_ = [("y", ctypes.c_void_p), ("y_pitch", ctypes.c_longlong), ("u", ctypes.c_void_p), ("v", ctypes.c_void_p),
                ("uv_pitch", ctypes.c_longlong), ("uv_step", ctypes.c_int), ("w", ctypes.c_int), ("h", ctypes.c_int)]


class StridedFrame(ctypes.Structure):
    """yfv2_strided_frame: channel k of pixel (r, c) at ch_k + r*pitch + c*step (RGB, BGRA / RGBA, grey, planar RGB)."""
    _fields_ = [("b", ctypes.c_void_p), ("g", ctypes.c_void_p), ("r", ctypes.c_void_p), ("pitch", ctypes.c_longlong),
                ("step", ctypes.c_int), ("w", ctypes.c_int), ("h", ctypes.c_int)]


class Yuv422Frame(ctypes.Structure):
    """yfv2_yuv422_frame: one packed YUV 4:2:2 source frame (YUYV / UYVY / YVYU) in device memory."""
    _fields_ = [("y", ctypes.c_void_p), ("u", ctypes.c_void_p), ("v", ctypes.c_void_p), ("pitch", ctypes.c_longlong),
                ("w", ctypes.c_int), ("h", ctypes.c_int)]


class TrainerOp(ctypes.Structure):
    """yfv2_trainer_op: one op of the native trainer's program (test hook)."""
    _fields_ = [(f, ctypes.c_int) for f in ("kind", "a", "b", "y", "pw", "pg", "pb", "pbias", "bn", "relu", "ks", "stride", "M")] + \
               [("aux", ctypes.c_longlong)]


class TrainerTensor(ctypes.Structure):
    """yfv2_trainer_tensor: where the trainer keeps one tensor and its gradient (test hook)."""
    _fields_ = [("off", ctypes.c_longlong), ("goff", ctypes.c_longlong), ("C", ctypes.c_int), ("H", ctypes.c_int), ("W", ctypes.c_int),
                ("ext", ctypes.c_int)]


TRAINER_OP_KINDS = ("stem", "bn", "pool", "pw", "dw", "up", "odd", "cate", "cat2")       # yfv2_trainer_op.kind
TRAINER_LAYOUT = ("ws_floats", "scratch_off", "pscratch_off", "pscratch_floats", "gflat_off", "gflat_floats", "wscratch_off",
                  "wscratch_floats")                                                     # yfv2_trainer_debug_layout


def trainer_program(handle):
    """(ops, tensors, layout) of a yfv2_trainer handle as lists of dicts / a dict; host only (test hook)."""
    L, n = lib(), ctypes.c_int()
    _check(L.yfv2_trainer_debug_ops(handle, None, 0, ctypes.byref(n)), "trainer_debug_ops")
    ops = (TrainerOp * n.value)()
    _check(L.yfv2_trainer_debug_ops(handle, ops, n.value, ctypes.byref(n)), "trainer_debug_ops")
    _check(L.yfv2_trainer_debug_tensors(handle, None, 0, ctypes.byref(n)), "trainer_debug_tensors")
    tens = (TrainerTensor * n.value)()
    _check(L.yfv2_trainer_debug_tensors(handle, tens, n.value, ctypes.byref(n)), "trainer_debug_tensors")
    lay = (ctypes.c_longlong * len(TRAINER_LAYOUT))()
    _check(L.yfv2_trainer_debug_layout(handle, lay), "trainer_debug_layout")
    as_dict = lambda s: {f: getattr(s, f) for f, _ in s._fields_}
    ops = [as_dict(o) for o in ops]
    for o in ops:
        o["kind"] = TRAINER_OP_KINDS[o["kind"]]
    return ops, [as_dict(t) for t in tens], dict(zip(TRAINER_LAYOUT, lay))


def check_bn_batch(N, H, W):
    """F.batch_norm in training mode refuses a layer with one value per channel; the deepest BatchNorm layers of the network run
    at stride 32 (stem 3x3 s2, max-pool 3x3 s2 p1 and three stride-2 blocks: each (h - 1) // 2 + 1), the first of them on the
    96 channels of stage4.0's projection branch.  Raised before anything is launched, as the reference raises at that layer."""
    h, w = H // 2, W // 2
    for _ in range(4):
        h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    if N * h * w == 1:
        raise ValueError("Expected more than 1 value per channel when training, got input size torch.Size([%d, 96, %d, %d])" % (N, h, w))


class Region(ctypes.Structure):
    """yfv2_region: a crop (x0, y0, w, h) of frame `frame` whose NMS rows yfv2_merge_regions maps back and merges."""
    _fields_ = [("frame", ctypes.c_int), ("x0", ctypes.c_int), ("y0", ctypes.c_int), ("w", ctypes.c_int), ("h", ctypes.c_int)]


# name -> (restype, argtypes); must list every prototype of include/yfv2.h (tests check this)
PROTOTYPES = {
    "yfv2_abi_version": (ctypes.c_int, []),
    "yfv2_last_error": (ctypes.c_char_p, []),
    "yfv2_plan_create": (ctypes.c_int, [_c_void_pp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                        ctypes.c_int, ctypes.c_int, ctypes.c_int]),
    "yfv2_plan_destroy": (ctypes.c_int, [ctypes.c_void_p]),
    "yfv2_plan_workspace_bytes": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_size_t)]),
    "yfv2_plan_invalidate_workspace": (ctypes.c_int, [ctypes.c_void_p]),
    "yfv2_plan_packed_bytes": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_size_t)]),
    "yfv2_plan_forward_launches": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int)]),
    "yfv2_pack_weights": (ctypes.c_int, [ctypes.c_void_p, _c_void_pp, _c_void_pp, ctypes.c_void_p, ctypes.c_void_p]),
    "yfv2_forward": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, _c_void_pp, ctypes.c_void_p,
                                    ctypes.c_void_p]),
    "yfv2_forward_u8": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, _c_void_pp, ctypes.c_void_p,
                                       ctypes.c_void_p]),
    "yfv2_decode": (ctypes.c_int, [_c_void_pp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                   ctypes.POINTER(ctypes.c_double), ctypes.c_void_p, ctypes.c_void_p]),
    "yfv2_export_heads": (ctypes.c_int, [_c_void_pp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                         ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "yfv2_nms_workspace_bytes": (ctypes.c_int, [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_size_t)]),
    "yfv2_nms": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_double,
                                ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_void_p,
                                ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "yfv2_decode_nms": (ctypes.c_int, [_c_void_pp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                       ctypes.POINTER(ctypes.c_double), ctypes.c_float, ctypes.c_double, ctypes.c_void_p,
                                       ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p,
                                       ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "yfv2_merge_regions": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(Region), ctypes.c_int, ctypes.c_int,
                                          ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.c_int, ctypes.c_int,
                                          ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "yfv2_batch_statistics": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                             ctypes.c_int, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p]),
    "yfv2_aug_contrast_brightness": (ctypes.c_int, [ctypes.c_void_p] * 4 + [ctypes.c_int, ctypes.c_longlong, ctypes.c_void_p]),
    "yfv2_resize_bgr_u8": (ctypes.c_int, [ctypes.POINTER(Frame), ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                          ctypes.c_void_p]),
    "yfv2_resize_yuv420_u8": (ctypes.c_int, [ctypes.POINTER(Yuv420Frame), ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                             ctypes.c_void_p]),
    "yfv2_resize_strided_u8": (ctypes.c_int, [ctypes.POINTER(StridedFrame), ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                              ctypes.c_void_p, ctypes.c_void_p]),
    "yfv2_resize_yuv422_u8": (ctypes.c_int, [ctypes.POINTER(Yuv422Frame), ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                             ctypes.c_void_p]),
    "yfv2_detect_u8_host": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                           ctypes.POINTER(ctypes.c_double), ctypes.c_float, ctypes.c_double, ctypes.c_int,
                                           ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "yfv2_detect_workspace_bytes": (ctypes.c_size_t, [ctypes.c_void_p, ctypes.c_int]),
    "yfv2_loss_workspace_bytes": (ctypes.c_int, [ctypes.c_int] * 6 + [ctypes.POINTER(ctypes.c_size_t)]),
    "yfv2_compute_loss": (ctypes.c_int, [_c_void_pp, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                         ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_double), ctypes.c_void_p, _c_void_pp,
                                         ctypes.c_void_p, ctypes.c_void_p]),
    "yfv2_loss_read_targets": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                              ctypes.c_int, ctypes.POINTER(ctypes.c_int), ctypes.c_void_p, ctypes.c_void_p,
                                              ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "yfv2_op_conv1x1_fwd": (ctypes.c_int, [ctypes.c_void_p] * 4 + [ctypes.c_int] * 4 + [ctypes.c_void_p]),
    "yfv2_op_conv1x1_bwd": (ctypes.c_int, [ctypes.c_void_p] * 6 + [ctypes.c_int] * 4 + [ctypes.c_void_p]),
    "yfv2_op_dwconv_fwd": (ctypes.c_int, [ctypes.c_void_p] * 3 + [ctypes.c_int] * 6 + [ctypes.c_void_p]),
    "yfv2_op_dwconv_bwd": (ctypes.c_int, [ctypes.c_void_p] * 5 + [ctypes.c_int] * 6 + [ctypes.c_void_p]),
    "yfv2_op_stem_fwd": (ctypes.c_int, [ctypes.c_void_p] * 3 + [ctypes.c_int] * 4 + [ctypes.c_void_p]),
    "yfv2_op_stem_wgrad": (ctypes.c_int, [ctypes.c_void_p] * 3 + [ctypes.c_int] * 4 + [ctypes.c_void_p]),
    "yfv2_op_bn_train_fwd": (ctypes.c_int, [ctypes.c_void_p] * 9 + [ctypes.c_int] * 4 + [ctypes.c_void_p]),
    "yfv2_op_bn_train_bwd": (ctypes.c_int, [ctypes.c_void_p] * 10 + [ctypes.c_int] * 4 + [ctypes.c_void_p]),
    "yfv2_op_maxpool_fwd": (ctypes.c_int, [ctypes.c_void_p] * 3 + [ctypes.c_int] * 3 + [ctypes.c_void_p]),
    "yfv2_op_maxpool_bwd": (ctypes.c_int, [ctypes.c_void_p] * 3 + [ctypes.c_int] * 3 + [ctypes.c_void_p]),
    "yfv2_op_upsample2_fwd": (ctypes.c_int, [ctypes.c_void_p] * 2 + [ctypes.c_int] * 3 + [ctypes.c_void_p]),
    "yfv2_op_upsample2_bwd": (ctypes.c_int, [ctypes.c_void_p] * 2 + [ctypes.c_int] * 3 + [ctypes.c_void_p]),
    "yfv2_trainer_create": (ctypes.c_int, [_c_void_pp] + [ctypes.c_int] * 6),
    "yfv2_trainer_destroy": (None, [ctypes.c_void_p]),
    "yfv2_trainer_workspace_bytes": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_size_t)]),
    "yfv2_trainer_grad_floats": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_longlong)]),
    "yfv2_trainer_param_offset": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_longlong), ctypes.POINTER(ctypes.c_longlong)]),
    "yfv2_train_forward": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, _c_void_pp, _c_void_pp, _c_void_pp, ctypes.c_void_p, ctypes.c_void_p]),
    "yfv2_train_backward": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, _c_void_pp, _c_void_pp, _c_void_pp, ctypes.c_void_p, ctypes.c_int,
                                           ctypes.c_void_p, ctypes.c_void_p]),
    "yfv2_trainer_debug_ops": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_int)]),
    "yfv2_trainer_debug_tensors": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_int)]),
    "yfv2_trainer_debug_layout": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_longlong)]),
    "yfv2_plan_stage_name": (ctypes.c_char_p, [ctypes.c_void_p, ctypes.c_int]),
    "yfv2_plan_stage_group": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int]),
    "yfv2_forward_range": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, _c_void_pp,
                                          ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    "yfv2_debug_pw_tc": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
                                        ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    "yfv2_debug_gather": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                                         ctypes.POINTER(ctypes.c_int), ctypes.c_void_p]),
    "yfv2_debug_nms_profile": (ctypes.c_int, [ctypes.c_void_p]),
    "yfv2_debug_heads_staged": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]),
    "yfv2_ncnn_post": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                      ctypes.POINTER(ctypes.c_float), ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_float,
                                      ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
}


def lib():
    """Loads libyfv2.so (once).  Raises if it has not been built — there is no fallback path."""
    global _lib
    if _lib is None:
        with _lock:
            if _lib is None:
                if not os.path.exists(_LIB_PATH):
                    raise RuntimeError("libyfv2.so is missing (%s): build it with "
                                       "`python yolo-fastestv2_b200/build.py` or __graft_entry__.build()" % _LIB_PATH)
                L = ctypes.CDLL(_LIB_PATH)
                for name, (res, args) in PROTOTYPES.items():
                    fn = getattr(L, name)
                    fn.restype, fn.argtypes = res, args
                _lib = L
    return _lib


class Yfv2Error(RuntimeError):
    pass


def _check(rc, what):
    if rc != 0:
        raise Yfv2Error("%s failed (%d): %s" % (what, rc, lib().yfv2_last_error().decode("utf-8", "replace")))


def _stream(device):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _ptr_array(tensors):
    arr = (ctypes.c_void_p * len(tensors))()
    for i, t in enumerate(tensors):
        arr[i] = t.data_ptr()
    return arr


def _require_cuda(t, name):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise Yfv2Error("%s must be a CUDA tensor: this implementation has no CPU path" % name)


class Trainer:
    """One yfv2_trainer (the native train-mode forward + backward of the whole network) with its workspace.  The workspace keeps
    ONE batch's activations: backward() must follow the forward() of the same batch."""

    def __init__(self, device, N, H, W, A, C):
        L = lib()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise Yfv2Error("trainers exist on CUDA devices only")
        self.N, self.H, self.W, self.A, self.C = N, H, W, A, C
        self._h = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            _check(L.yfv2_trainer_create(ctypes.byref(self._h), self.device.index or 0, N, H, W, A, C), "trainer_create")
        nb = ctypes.c_size_t()
        _check(L.yfv2_trainer_workspace_bytes(self._h, ctypes.byref(nb)), "trainer_workspace_bytes")
        self.workspace = torch.empty(nb.value, dtype=torch.uint8, device=self.device)
        n = ctypes.c_longlong()
        _check(L.yfv2_trainer_grad_floats(self._h, ctypes.byref(n)), "trainer_grad_floats")
        self.grad_floats = n.value
        self.param_offsets = []
        off, num = ctypes.c_longlong(), ctypes.c_longlong()
        for i in range(225):
            _check(L.yfv2_trainer_param_offset(self._h, i, ctypes.byref(off), ctypes.byref(num)), "trainer_param_offset")
            self.param_offsets.append((off.value, num.value))
        self.generation = 0                  # bumped by every forward: a backward must see the generation of its own forward
        # persistent buffers: the C side replays its two programs as CUDA graphs while every pointer stays the same
        self.x_static = torch.empty((N, 3, H, W), dtype=torch.float32, device=self.device)
        self.preds_static = self.alloc_preds()
        self.dpreds_static = [torch.empty_like(p) for p in self.preds_static]
        self.flat_static = torch.empty(self.grad_floats, dtype=torch.float32, device=self.device)

    def __del__(self):
        try:
            if getattr(self, "_h", None) is not None and self._h.value:
                lib().yfv2_trainer_destroy(self._h)
                self._h = ctypes.c_void_p()
        except Exception:
            pass

    def program(self):
        """(ops, tensors, layout) of the trainer's static program (trainer_program; host only)."""
        return trainer_program(self._h)

    def alloc_preds(self):
        out = []
        for s in (16, 32):
            h, w = self.H // s, self.W // s
            for ch in (4 * self.A, self.A, self.C):
                out.append(torch.empty((self.N, ch, h, w), dtype=torch.float32, device=self.device))
        return out

    @staticmethod
    def _check_weights(params, bn_running):
        if len(params) != 225 or len(bn_running) != 146:
            raise Yfv2Error("trainer: expected 225 parameters and 146 BN buffers, got %d / %d" % (len(params), len(bn_running)))
        for t in list(params) + list(bn_running):
            _require_cuda(t, "weight")
            if t.dtype != torch.float32 or not t.is_contiguous():
                raise Yfv2Error("trainer: weights must be contiguous float32")

    def forward(self, x, params, bn_running):
        self._check_weights(params, bn_running)
        _require_cuda(x, "x")
        if tuple(x.shape) != (self.N, 3, self.H, self.W) or x.dtype != torch.float32 or not x.is_contiguous():
            raise Yfv2Error("trainer: expected a contiguous float32 input of shape %s" % ((self.N, 3, self.H, self.W),))
        self.x_static.copy_(x)                               # (the graph reads the batch from a fixed address)
        preds = self.preds_static
        with torch.cuda.device(self.device):
            _check(lib().yfv2_train_forward(self._h, ctypes.c_void_p(self.x_static.data_ptr()), _ptr_array(params), _ptr_array(bn_running),
                                            _ptr_array(preds), ctypes.c_void_p(self.workspace.data_ptr()), _stream(self.device)),
                   "train_forward")
        self.generation += 1
        return [p.detach() for p in preds]                   # aliases of the trainer's head buffers (overwritten by the next forward)

    def backward(self, params, dpreds, grads_flat, accumulate):
        """Backward of the last forward().  grads_flat None: the trainer's own flat buffer (overwritten) is used and returned."""
        if grads_flat is None:
            grads_flat, accumulate = self.flat_static, False
        if grads_flat.numel() != self.grad_floats or grads_flat.dtype != torch.float32 or not grads_flat.is_contiguous():
            raise Yfv2Error("trainer: grads_flat must be a contiguous float32 buffer of %d elements" % self.grad_floats)
        torch._foreach_copy_(self.dpreds_static, [d if d.is_contiguous() else d.contiguous() for d in dpreds])
        with torch.cuda.device(self.device):
            _check(lib().yfv2_train_backward(self._h, ctypes.c_void_p(self.x_static.data_ptr()), _ptr_array(params),
                                             _ptr_array(self.preds_static), _ptr_array(self.dpreds_static),
                                             ctypes.c_void_p(grads_flat.data_ptr()), int(bool(accumulate)),
                                             ctypes.c_void_p(self.workspace.data_ptr()), _stream(self.device)), "train_backward")
        return grads_flat


def anchors_array(cfg):
    a = [float(v) for v in cfg["anchors"]]
    return (ctypes.c_double * len(a))(*a)


class Plan:
    """One yfv2_plan with its workspace and packed-weight buffer (owned here as torch tensors)."""

    def __init__(self, device, N, H, W, A, C, training=False, detect_max_det=0):
        L = lib()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise Yfv2Error("plans exist on CUDA devices only")
        self.N, self.H, self.W, self.A, self.C = N, H, W, A, C
        self._h = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            _check(L.yfv2_plan_create(ctypes.byref(self._h), self.device.index or 0, N, H, W, A, C, int(training)), "plan_create")
        nb = ctypes.c_size_t()
        _check(L.yfv2_plan_workspace_bytes(self._h, ctypes.byref(nb)), "workspace_bytes")
        ws_bytes = nb.value
        if detect_max_det:
            ws_bytes = max(ws_bytes, L.yfv2_detect_workspace_bytes(self._h, detect_max_det))
        self.workspace = torch.empty(ws_bytes, dtype=torch.uint8, device=self.device)
        _check(L.yfv2_plan_packed_bytes(self._h, ctypes.byref(nb)), "packed_bytes")
        self.packed = torch.empty(nb.value, dtype=torch.uint8, device=self.device)
        n = ctypes.c_int()
        _check(L.yfv2_plan_forward_launches(self._h, ctypes.byref(n)), "forward_launches")
        self.forward_launches = n.value
        self.stage_names = []                 # fused stages; stages sharing a stage_groups value are one kernel launch
        while True:
            nm = L.yfv2_plan_stage_name(self._h, len(self.stage_names))
            if nm is None:
                break
            self.stage_names.append(nm.decode())
        self.stage_groups = [L.yfv2_plan_stage_group(self._h, i) for i in range(len(self.stage_names))]
        self.packed_version = None

    def __del__(self):
        try:
            if getattr(self, "_h", None) is not None and self._h.value:
                lib().yfv2_plan_destroy(self._h)
                self._h = ctypes.c_void_p()
        except Exception:
            pass

    def pack(self, params, bn_running):
        """params: 225 fp32 CUDA tensors in Detector.parameters() order; bn_running: 146 (mean, var, ...)."""
        if len(params) != 225 or len(bn_running) != 146:
            raise Yfv2Error("pack: expected 225 parameters and 146 BN buffers, got %d / %d" % (len(params), len(bn_running)))
        keep = []
        for t in list(params) + list(bn_running):
            _require_cuda(t, "weight")
            if t.dtype != torch.float32:
                raise Yfv2Error("weights must be float32")
            keep.append(t.detach().contiguous())
        with torch.cuda.device(self.device):
            _check(lib().yfv2_pack_weights(self._h, _ptr_array(keep[:225]), _ptr_array(keep[225:]),
                                           ctypes.c_void_p(self.packed.data_ptr()), _stream(self.device)), "pack_weights")
        return keep   # caller may drop it after the stream has run; kept alive by stream ordering of the allocator

    def alloc_preds(self):
        N, A, C = self.N, self.A, self.C
        out = []
        for s in (16, 32):
            h, w = self.H // s, self.W // s
            for ch in (4 * A, A, C):
                out.append(torch.empty((N, ch, h, w), dtype=torch.float32, device=self.device))
        return tuple(out)

    def forward(self, x, preds=None):
        _require_cuda(x, "x")
        if tuple(x.shape) != (self.N, 3, self.H, self.W):
            raise Yfv2Error("forward: input shape %s does not match the plan (%d,3,%d,%d)" % (tuple(x.shape), self.N, self.H, self.W))
        if x.dtype not in (torch.float32, torch.uint8):
            raise Yfv2Error("forward: input must be float32 or uint8")
        x = x.contiguous()
        if preds is None:
            preds = self.alloc_preds()
        fn = lib().yfv2_forward if x.dtype == torch.float32 else lib().yfv2_forward_u8
        with torch.cuda.device(self.device):
            _check(fn(self._h, ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(self.packed.data_ptr()), _ptr_array(preds),
                      ctypes.c_void_p(self.workspace.data_ptr()), _stream(self.device)), "forward")
        return preds

    def forward_range(self, x, preds, first, last):
        """Runs fused stages [first,last) only (see yfv2.h); x, preds as in forward()."""
        with torch.cuda.device(self.device):
            _check(lib().yfv2_forward_range(self._h, ctypes.c_void_p(x.data_ptr()), int(x.dtype == torch.uint8),
                                            ctypes.c_void_p(self.packed.data_ptr()), _ptr_array(preds),
                                            ctypes.c_void_p(self.workspace.data_ptr()), first, last, _stream(self.device)),
                   "forward_range")

    def debug_gather(self, which):
        """Dense NCHW copy of an intermediate tensor of the last forward (test hook, see yfv2.h)."""
        dims = (ctypes.c_int * 4)()
        _check(lib().yfv2_debug_gather(self._h, ctypes.c_void_p(self.workspace.data_ptr()), which, None, dims, None), "debug_gather")
        out = torch.empty(tuple(dims), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            _check(lib().yfv2_debug_gather(self._h, ctypes.c_void_p(self.workspace.data_ptr()), which,
                                           ctypes.c_void_p(out.data_ptr()), dims, _stream(self.device)), "debug_gather")
        return out

    def detect_u8_host(self, x_host, anchors, conf_thres, iou_thres, out_host, counts_host, max_det=MAX_DET):
        """Whole step from pinned host uint8 images to pinned host detections (asynchronous)."""
        with torch.cuda.device(self.device):
            _check(lib().yfv2_detect_u8_host(self._h, ctypes.c_void_p(x_host.data_ptr()), ctypes.c_void_p(self.packed.data_ptr()),
                                             anchors, ctypes.c_float(conf_thres), ctypes.c_double(iou_thres), max_det,
                                             ctypes.c_void_p(out_host.data_ptr()), ctypes.c_void_p(counts_host.data_ptr()),
                                             ctypes.c_void_p(self.workspace.data_ptr()), _stream(self.device)), "detect_u8_host")


def decode(preds, cfg):
    """handel_preds on the device: returns [N, M, 5+C] fp32 CUDA tensor."""
    for p in preds:
        _require_cuda(p, "preds")
    preds = [p.detach().contiguous().float() for p in preds]
    N, A4, h, w = preds[0].shape
    A, C = preds[1].shape[1], preds[2].shape[1]
    if len(preds) != 6 or A4 != 4 * A:
        raise Yfv2Error("decode: expected the 6-tuple (reg,obj,cls) x 2 levels")
    H, W = h * 16, w * 16
    if cfg is not None and (int(cfg["height"]) != H or int(cfg["width"]) != W):
        raise Yfv2Error("decode: head tensors are %dx%d/16 but cfg says %sx%s" % (H, W, cfg["height"], cfg["width"]))
    M = (h * w + preds[3].shape[2] * preds[3].shape[3]) * A
    out = torch.empty((N, M, 5 + C), dtype=torch.float32, device=preds[0].device)
    with torch.cuda.device(out.device):
        _check(lib().yfv2_decode(_ptr_array(preds), N, H, W, A, C, anchors_array(cfg), ctypes.c_void_p(out.data_ptr()),
                                 _stream(out.device)), "decode")
    return out


def _filter_tensor(classes, device):
    if classes is None:
        return None, 0
    classes = list(classes)
    if not classes:
        classes = [-1]      # the reference keeps rows whose class is IN the list (utils/utils.py:266-268): an empty list keeps nothing
    t = torch.as_tensor(classes, dtype=torch.int32, device=device)
    return t, t.numel()


def nms(dets, conf_thres=0.3, iou_thres=0.45, classes=None, max_det=MAX_DET, want_idx=True, max_wh=MAX_WH):
    """Device NMS.  Returns (out [N,max_det,6], counts [N] int32, kept_idx [N,max_det] int32 or None).
    max_wh: the per-class box offset of utils/utils.py:283."""
    _require_cuda(dets, "dets")
    dets = dets.detach().contiguous().float()
    N, M, D = dets.shape
    out = torch.empty((N, max_det, 6), dtype=torch.float32, device=dets.device)
    counts = torch.empty((N,), dtype=torch.int32, device=dets.device)
    idx = torch.empty((N, max_det), dtype=torch.int32, device=dets.device) if want_idx else None
    filt, nf = _filter_tensor(classes, dets.device)
    with torch.cuda.device(dets.device):
        _check(lib().yfv2_nms(ctypes.c_void_p(dets.data_ptr()), N, M, D - 5, ctypes.c_float(conf_thres), ctypes.c_double(iou_thres),
                              ctypes.c_void_p(filt.data_ptr()) if nf else None, nf, max_det, ctypes.c_float(max_wh),
                              ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(counts.data_ptr()),
                              ctypes.c_void_p(idx.data_ptr()) if want_idx else None, None, _stream(dets.device)), "nms")
    return out, counts, idx


def decode_nms(preds, cfg, conf_thres=0.3, iou_thres=0.45, classes=None, max_det=MAX_DET, want_idx=False, max_wh=MAX_WH):
    """Fused handel_preds + non_max_suppression on the device (no [N,M,5+C] tensor)."""
    for p in preds:
        _require_cuda(p, "preds")
    preds = [p.detach().contiguous().float() for p in preds]
    N, _, h, w = preds[0].shape
    A, C = preds[1].shape[1], preds[2].shape[1]
    H, W = h * 16, w * 16
    dev = preds[0].device
    out = torch.empty((N, max_det, 6), dtype=torch.float32, device=dev)
    counts = torch.empty((N,), dtype=torch.int32, device=dev)
    idx = torch.empty((N, max_det), dtype=torch.int32, device=dev) if want_idx else None
    filt, nf = _filter_tensor(classes, dev)
    with torch.cuda.device(dev):
        _check(lib().yfv2_decode_nms(_ptr_array(preds), N, H, W, A, C, anchors_array(cfg), ctypes.c_float(conf_thres),
                                     ctypes.c_double(iou_thres), ctypes.c_void_p(filt.data_ptr()) if nf else None, nf, max_det,
                                     ctypes.c_float(max_wh), ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(counts.data_ptr()),
                                     ctypes.c_void_p(idx.data_ptr()) if want_idx else None, None, _stream(dev)), "decode_nms")
    return out, counts, idx


MERGE_METRICS = {"iou": 0, "ios": 1}


def merge_regions(dets, counts, regions, F, W, H, thr, metric, max_det):
    """yfv2_merge_regions: the NMS rows of T region images -> one list per frame in frame pixels (a cross-region NMS, see
    include/yfv2.h).  dets: CUDA float32 [T, max_det_in, 6] and counts int32 [T], as decode_nms / nms return them for the region
    images; regions: T tuples (frame, x0, y0, w, h), the regions of one frame contiguous, frames ascending; F frames; W x H the
    network input the regions were stretched to; metric "iou" | "ios" (or 0 | 1).  Returns CUDA tensors (out float64
    [F, max_det, 6], counts int32 [F], kept_src int32 [F, max_det]: t * max_det_in + row of each kept row, -1 past the count)."""
    _require_cuda(dets, "dets")
    _require_cuda(counts, "counts")
    if dets.dim() != 3 or dets.shape[2] != 6 or dets.dtype != torch.float32:
        raise Yfv2Error("merge_regions: dets must be float32 [T, max_det_in, 6], got %s %s" % (dets.dtype, tuple(dets.shape)))
    T, max_det_in = dets.shape[0], dets.shape[1]
    if counts.dtype != torch.int32 or tuple(counts.shape) != (T,):
        raise Yfv2Error("merge_regions: counts must be int32 [%d], got %s %s" % (T, counts.dtype, tuple(counts.shape)))
    regions = list(regions)
    if len(regions) != T:
        raise Yfv2Error("merge_regions: %d regions for %d row blocks" % (len(regions), T))
    m = MERGE_METRICS.get(metric, metric)
    if m not in (0, 1):
        raise Yfv2Error("merge_regions: metric must be 'iou' or 'ios', got %r" % (metric,))
    dets, counts = dets.contiguous(), counts.contiguous()
    descs = (Region * max(T, 1))()
    for d, r in zip(descs, regions):
        d.frame, d.x0, d.y0, d.w, d.h = (int(v) for v in r)
    dev = dets.device
    out = torch.empty((max(F, 0), max_det, 6), dtype=torch.float64, device=dev)
    out_counts = torch.empty((max(F, 0),), dtype=torch.int32, device=dev)
    kept = torch.empty((max(F, 0), max_det), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _check(lib().yfv2_merge_regions(ctypes.c_void_p(dets.data_ptr()), ctypes.c_void_p(counts.data_ptr()), descs, T, max_det_in, F,
                                        H, W, ctypes.c_double(thr), m, max_det, ctypes.c_void_p(out.data_ptr()),
                                        ctypes.c_void_p(out_counts.data_ptr()), ctypes.c_void_p(kept.data_ptr()), _stream(dev)),
               "merge_regions")
    return out, out_counts, kept


def batch_statistics(out, counts, targets, iou_threshold):
    """True-positive flags [N,max_det] (float 0/1) of NMS output rows against pixel-xyxy targets [nt,6] (device)."""
    _require_cuda(out, "out")
    N, max_det, _ = out.shape
    targets = targets.detach().to(out.device).float().contiguous().reshape(-1, 6)
    tp = torch.empty((N, max_det), dtype=torch.float32, device=out.device)
    with torch.cuda.device(out.device):
        _check(lib().yfv2_batch_statistics(ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(counts.data_ptr()), N, max_det,
                                           ctypes.c_void_p(targets.data_ptr()) if targets.numel() else None, targets.shape[0],
                                           ctypes.c_float(iou_threshold), ctypes.c_void_p(tp.data_ptr()), _stream(out.device)),
               "batch_statistics")
    return tp


def contrast_and_brightness(imgs, alpha, beta, out=None):
    """utils.datasets.contrast_and_brightness (cv2.addWeighted on uint8) for a batch on the device: imgs uint8 [N, ...],
    alpha / beta float32 [N] (one pair per image).  Returns a new uint8 tensor (or writes `out`, which may be `imgs`)."""
    _require_cuda(imgs, "imgs")
    if imgs.dtype != torch.uint8:
        raise TypeError("contrast_and_brightness expects uint8 images (the reference augments before the /255)")
    imgs = imgs.contiguous()
    N = imgs.shape[0]
    alpha = torch.as_tensor(alpha, dtype=torch.float32).to(imgs.device).contiguous().reshape(-1)
    beta = torch.as_tensor(beta, dtype=torch.float32).to(imgs.device).contiguous().reshape(-1)
    if alpha.numel() != N or beta.numel() != N:
        raise ValueError("one (alpha, beta) pair per image")
    if out is None:
        out = torch.empty_like(imgs)
    with torch.cuda.device(imgs.device):
        _check(lib().yfv2_aug_contrast_brightness(ctypes.c_void_p(imgs.data_ptr()), ctypes.c_void_p(out.data_ptr()),
                                                  ctypes.c_void_p(alpha.data_ptr()), ctypes.c_void_p(beta.data_ptr()), N,
                                                  imgs.numel() // N, _stream(imgs.device)), "aug_contrast_brightness")
    return out


def _frame_on_device(f, device):
    """A packed HWC BGR uint8 frame as a CUDA tensor on `device` whose pixels are 3 bytes apart (rows may be further apart)."""
    if not isinstance(f, torch.Tensor):
        import numpy as np
        f = torch.from_numpy(np.ascontiguousarray(f))
    if f.dtype != torch.uint8 or f.dim() != 3 or f.shape[2] != 3:
        raise Yfv2Error("resize_bgr: frames must be uint8 [h, w, 3] (BGR, as cv2.imread returns), got %s %s"
                        % (f.dtype, tuple(f.shape)))
    f = f.to(device)
    if f.stride(2) != 1 or f.stride(1) != 3:
        f = f.contiguous()
    return f


def resize_bgr(frames, W, H, device=None, out=None):
    """cv2.resize(frame, (W, H), interpolation=cv2.INTER_LINEAR) of every frame, transposed to the [N, 3, H, W] uint8 batch the
    network takes (test.py:34-37), bit for bit, in one kernel.  frames: HWC uint8 BGR numpy arrays or CUDA tensors, any sizes
    (host arrays are copied to `device` first; a CUDA tensor that is a row crop of a larger frame is read in place)."""
    frames = list(frames)
    if not frames:
        raise Yfv2Error("resize_bgr: no frames")
    if device is None:
        cuda = [f.device for f in frames if isinstance(f, torch.Tensor) and f.is_cuda]
        device = cuda[0] if cuda else torch.device("cuda", torch.cuda.current_device())
    device = torch.device(device)
    if device.type != "cuda":
        raise Yfv2Error("resize_bgr: runs on CUDA devices only (no CPU fallback)")
    dev_frames = [_frame_on_device(f, device) for f in frames]
    descs = (Frame * len(dev_frames))()
    for d, f in zip(descs, dev_frames):
        d.data, d.w, d.h, d.pitch = f.data_ptr(), f.shape[1], f.shape[0], f.stride(0)
    N = len(dev_frames)
    if out is None:
        out = torch.empty((N, 3, H, W), dtype=torch.uint8, device=device)
    elif tuple(out.shape) != (N, 3, H, W) or out.dtype != torch.uint8 or not out.is_contiguous() or out.device != device:
        raise Yfv2Error("resize_bgr: out must be a contiguous uint8 tensor of shape %s on %s" % ((N, 3, H, W), device))
    with torch.cuda.device(device):
        _check(lib().yfv2_resize_bgr_u8(descs, N, H, W, ctypes.c_void_p(out.data_ptr()), _stream(device)), "resize_bgr_u8")
    return out


YUV420_LAYOUTS = ("nv12", "nv21", "i420", "yv12")


def _uint8_plane(p, what):
    """p as a uint8 2-D torch tensor; a host numpy array is wrapped, not copied."""
    if not isinstance(p, torch.Tensor):
        import numpy as np
        p = np.asarray(p)
        if p.dtype != np.uint8 or p.ndim != 2:
            raise Yfv2Error("resize_yuv420: %s must be a uint8 2-D array, got %s %s" % (what, p.dtype, p.shape))
        p = torch.from_numpy(p if min(p.strides, default=0) >= 0 else np.ascontiguousarray(p))
    elif p.dtype != torch.uint8 or p.dim() != 2:
        raise Yfv2Error("resize_yuv420: %s must be a uint8 2-D tensor, got %s %s" % (what, p.dtype, tuple(p.shape)))
    return p


def _yuv420_planes(f, layout, i):
    """Frame i as (y, u, v) uint8 2-D planes (u and v are the same [h/2, w] UV or VU plane for NV12 / NV21), checked, not
    copied.  A single buffer is cv2's [h*3/2, w] layout: the luma rows, then the chroma (interleaved rows for NV12 / NV21; for
    I420 / YV12 the two w/2-wide planes back to back, read from a contiguous buffer)."""
    interleaved = layout in ("nv12", "nv21")
    if isinstance(f, (tuple, list)):
        planes = [_uint8_plane(p, "frame %d plane %d" % (i, k)) for k, p in enumerate(f)]
        if len(planes) != (2 if interleaved else 3):
            raise Yfv2Error("resize_yuv420: frame %d: %s takes %s, got %d planes"
                            % (i, layout, "(y, uv)" if interleaved else "(y, u, v)", len(planes)))
        y = planes[0]
        h, w = y.shape
        chroma = [(h // 2, w)] if interleaved else [(h // 2, w // 2)] * 2
        for k, (p, want) in enumerate(zip(planes[1:], chroma)):
            if tuple(p.shape) != want or h % 2 or w % 2:
                raise Yfv2Error("resize_yuv420: frame %d: y %s needs even sizes and chroma planes of %s, plane %d is %s"
                                % (i, tuple(y.shape), want, k + 1, tuple(p.shape)))
        u, v = (planes[1], planes[1]) if interleaved else (planes[1], planes[2])
        return y, u, v
    buf = _uint8_plane(f, "frame %d" % i)
    rows, w = buf.shape
    h = rows // 3 * 2
    if rows % 3 or h <= 0 or w <= 0 or w % 2:
        raise Yfv2Error("resize_yuv420: frame %d: a single buffer is [h*3/2, w] with h, w even and > 0, got %s"
                        % (i, tuple(buf.shape)))
    if interleaved:
        return buf[:h], buf[h:], buf[h:]
    buf = buf.contiguous()
    flat, q = buf.reshape(-1), (h // 2) * (w // 2)
    first, second = (flat[h * w:h * w + q].view(h // 2, w // 2), flat[h * w + q:h * w + 2 * q].view(h // 2, w // 2))
    return (buf[:h],) + ((first, second) if layout == "i420" else (second, first))


def resize_yuv420(frames, W, H, layout, device=None, out=None):
    """cv2.resize(cv2.cvtColor(frame, cv2.COLOR_YUV2BGR_<LAYOUT>), (W, H), interpolation=cv2.INTER_LINEAR) of every frame,
    transposed to the [N, 3, H, W] uint8 batch the network takes, bit for bit, in one kernel (yfv2_resize_yuv420_u8).
    layout: "nv12" | "nv21" | "i420" | "yv12", or a list of one per frame (one launch may mix layouts).  Each frame is cv2's
    single uint8 buffer [h*3/2, w], or its planes: (y [h, w], uv [h/2, w]) for NV12 / NV21, (y, u [h/2, w/2], v [h/2, w/2]) for
    I420 / YV12; numpy arrays or CUDA tensors, any even sizes.  Planes may be views into larger surfaces (rows further apart than
    w): CUDA views are read in place, host arrays are copied to `device` (1.5 bytes per pixel)."""
    frames = list(frames)
    layouts = [layout] * len(frames) if isinstance(layout, str) else list(layout)
    for lay in layouts if layouts else [layout]:
        if lay not in YUV420_LAYOUTS:
            raise Yfv2Error("resize_yuv420: layout must be one of %s, got %r" % (", ".join(YUV420_LAYOUTS), lay))
    if not frames:
        raise Yfv2Error("resize_yuv420: no frames")
    if len(layouts) != len(frames):
        raise Yfv2Error("resize_yuv420: %d layouts for %d frames" % (len(layouts), len(frames)))
    planes = [_yuv420_planes(f, lay, i) for i, (f, lay) in enumerate(zip(frames, layouts))]
    if device is None:
        cuda = [p.device for ps in planes for p in ps if p.is_cuda]
        device = cuda[0] if cuda else torch.device("cuda", torch.cuda.current_device())
    device = torch.device(device)
    if device.type != "cuda":
        raise Yfv2Error("resize_yuv420: runs on CUDA devices only (no CPU fallback)")
    N = len(frames)
    if out is None:
        out = torch.empty((N, 3, H, W), dtype=torch.uint8, device=device)
    elif tuple(out.shape) != (N, 3, H, W) or out.dtype != torch.uint8 or not out.is_contiguous() or out.device != device:
        raise Yfv2Error("resize_yuv420: out must be a contiguous uint8 tensor of shape %s on %s" % ((N, 3, H, W), device))

    def on_device(p):
        p = p.to(device)
        return p if p.stride(1) == 1 else p.contiguous()

    descs = (Yuv420Frame * N)()
    keep = []          # device copies stay referenced until the launch is queued: a freed block could take the next frame's copy
    for d, (y, u, v), lay in zip(descs, planes, layouts):
        if lay in ("nv12", "nv21"):
            y, uv = on_device(y), on_device(u)
            keep += [y, uv]
            d.u = uv.data_ptr() + (lay == "nv21")
            d.v = uv.data_ptr() + (lay == "nv12")
            d.uv_pitch, d.uv_step = uv.stride(0), 2
        else:
            y, u, v = on_device(y), on_device(u), on_device(v)
            if u.stride(0) != v.stride(0):                 # one chroma pitch per descriptor
                u, v = u.contiguous(), v.contiguous()
            keep += [y, u, v]
            d.u, d.v, d.uv_pitch, d.uv_step = u.data_ptr(), v.data_ptr(), u.stride(0), 1
        d.y, d.y_pitch, d.h, d.w = y.data_ptr(), y.stride(0), y.shape[0], y.shape[1]
    with torch.cuda.device(device):
        _check(lib().yfv2_resize_yuv420_u8(descs, N, H, W, ctypes.c_void_p(out.data_ptr()), _stream(device)), "resize_yuv420_u8")
    return out


# Layouts yfv2_resize_strided_u8 takes: the byte offsets of B, G, R within a pixel of each packed one, and the number of bytes
# per pixel of each packed one.  "rgb_chw" ([3, h, w], R plane first) is built from its channel stride instead.
STRIDED_LAYOUTS = ("rgb", "bgra", "rgba", "gray", "rgb_chw")
_BGR_OFFSETS = {"rgb": (2, 1, 0), "bgra": (0, 1, 2), "rgba": (2, 1, 0), "gray": (0, 0, 0)}
# packed YUV 4:2:2 (yfv2_resize_yuv422_u8): the byte offsets of the first Y, of U and of V within a 4-byte macropixel
YUV422_LAYOUTS = ("yuyv", "uyvy", "yvyu")
_YUV422_OFFSETS = {"yuyv": (0, 1, 3), "uyvy": (1, 0, 2), "yvyu": (0, 3, 1)}
_CHANNELS = {"rgb": 3, "bgra": 4, "rgba": 4, "yuyv": 2, "uyvy": 2, "yvyu": 2}
LAYOUTS = ("bgr",) + YUV420_LAYOUTS + STRIDED_LAYOUTS + YUV422_LAYOUTS
# the entry point (descriptor kind) of each layout
_KIND = dict([("bgr", "bgr")] + [(k, "yuv420") for k in YUV420_LAYOUTS] + [(k, "strided") for k in STRIDED_LAYOUTS]
             + [(k, "yuv422") for k in YUV422_LAYOUTS])


def frame_size(frame, layout):
    """(h, w) in pixels of a frame in the given layout, as resize_frames takes it."""
    if layout in YUV420_LAYOUTS:
        if isinstance(frame, (tuple, list)):
            return tuple(frame[0].shape[:2])
        return frame.shape[0] // 3 * 2, frame.shape[1]
    return tuple(frame.shape[1:3]) if layout == "rgb_chw" else tuple(frame.shape[:2])


def _layout_frame(f, layout, i):
    """Frame i of a strided or 4:2:2 layout as a uint8 tensor of the layout's shape, checked, not copied."""
    shape = ("[3, h, w]" if layout == "rgb_chw" else "[h, w]" if layout == "gray" else "[h, w, %d]" % _CHANNELS[layout])
    if not isinstance(f, torch.Tensor):
        import numpy as np
        f = np.asarray(f)
        if f.dtype != np.uint8:
            raise Yfv2Error("resize_frames: frame %d (%s) must be uint8 %s, got %s %s" % (i, layout, shape, f.dtype, f.shape))
        f = torch.from_numpy(f if min(f.strides, default=0) >= 0 else np.ascontiguousarray(f))
    ok = f.dtype == torch.uint8 and f.dim() == (2 if layout == "gray" else 3) and f.numel() > 0
    if ok and layout == "rgb_chw":
        ok = f.shape[0] == 3
    elif ok and layout != "gray":
        ok = f.shape[2] == _CHANNELS[layout]
    if not ok:
        raise Yfv2Error("resize_frames: frame %d (%s) must be uint8 %s with h, w > 0, got %s %s"
                        % (i, layout, shape, f.dtype, tuple(f.shape)))
    if layout in YUV422_LAYOUTS and f.shape[1] % 2:
        raise Yfv2Error("resize_frames: frame %d (%s): 4:2:2 needs an even width (two pixels per macropixel), got w = %d"
                        % (i, layout, f.shape[1]))
    return f


def _check_frame(f, layout, i):
    """Checks frame i against its layout without launching anything; returns what the layout's resize takes."""
    kind = _KIND[layout]
    if kind == "bgr":
        if isinstance(f, torch.Tensor):
            ok = f.dtype == torch.uint8
        else:
            import numpy as np
            f = np.asarray(f)
            ok = f.dtype == np.uint8
        if not ok or f.ndim != 3 or f.shape[2] != 3:
            raise Yfv2Error("resize_frames: frame %d (bgr) must be uint8 [h, w, 3], got %s %s" % (i, f.dtype, tuple(f.shape)))
        return f
    if kind == "yuv420":
        _yuv420_planes(f, layout, i)
        return f
    return _layout_frame(f, layout, i)


def _resize_layout_run(frames, layouts, W, H, device, out):
    """One yfv2_resize_strided_u8 or yfv2_resize_yuv422_u8 call for checked frames of one descriptor kind."""
    N = len(frames)
    strided = _KIND[layouts[0]] == "strided"
    descs = ((StridedFrame if strided else Yuv422Frame) * N)()
    keep = []          # device copies stay referenced until the launch is queued: a freed block could take the next frame's copy
    for d, f, lay in zip(descs, frames, layouts):
        f = f.to(device)
        if lay == "rgb_chw":                                 # any channel and row stride, unit column stride
            if f.stride(2) != 1 or f.stride(1) < f.shape[2]:
                f = f.contiguous()
            p, s = f.data_ptr(), f.stride(0)
            d.b, d.g, d.r, d.pitch, d.step = p + 2 * s, p + s, p, f.stride(1), 1
            d.h, d.w = f.shape[1], f.shape[2]
        else:
            step = 1 if lay == "gray" else _CHANNELS[lay]
            if f.stride(1) != step or (lay != "gray" and f.stride(2) != 1) or f.stride(0) < step * f.shape[1]:
                f = f.contiguous()
            p = f.data_ptr()
            if strided:
                ob, og, or_ = _BGR_OFFSETS[lay]
                d.b, d.g, d.r, d.step = p + ob, p + og, p + or_, step
            else:
                oy, ou, ov = _YUV422_OFFSETS[lay]
                d.y, d.u, d.v = p + oy, p + ou, p + ov
            d.pitch, d.h, d.w = f.stride(0), f.shape[0], f.shape[1]
        keep.append(f)
    fn, what = ((lib().yfv2_resize_strided_u8, "resize_strided_u8") if strided else
                (lib().yfv2_resize_yuv422_u8, "resize_yuv422_u8"))
    with torch.cuda.device(device):
        _check(fn(descs, N, H, W, ctypes.c_void_p(out.data_ptr()), _stream(device)), what)


def resize_frames(frames, W, H, layout, device=None, out=None):
    """cv2.resize(cv2.cvtColor(frame, code), (W, H), interpolation=cv2.INTER_LINEAR) of every frame, transposed to the
    [N, 3, H, W] uint8 batch the network takes, bit for bit, for every frame layout the library reads.  layout: one name, or a
    list with one name per frame (one batch may mix layouts and sizes):
      "bgr"                             [h, w, 3], no conversion (as resize_bgr)
      "nv12" | "nv21" | "i420" | "yv12" cv2's [h*3/2, w] buffer or its planes, COLOR_YUV2BGR_<LAYOUT> (as resize_yuv420)
      "rgb"                             [h, w, 3], COLOR_RGB2BGR
      "bgra" | "rgba"                   [h, w, 4], COLOR_BGRA2BGR / COLOR_RGBA2BGR (alpha ignored)
      "gray"                            [h, w], COLOR_GRAY2BGR
      "rgb_chw"                         [3, h, w] planar RGB (torchvision's decode_jpeg): transpose + COLOR_RGB2BGR
      "yuyv" | "uyvy" | "yvyu"          [h, w, 2] packed 4:2:2 (w even), COLOR_YUV2BGR_<LAYOUT>
    Frames are numpy arrays or CUDA tensors; CUDA views with larger row strides or crop offsets are read in place (for
    "rgb_chw" any channel and row stride with unit column stride), host arrays are copied to `device`.  Consecutive frames of
    one descriptor kind go to one call (yfv2_resize_bgr_u8 / _yuv420_u8 / _strided_u8 / _yuv422_u8), each into its slice of
    `out`.  Every frame is checked before anything is copied or launched."""
    frames = list(frames)
    layouts = [layout] * len(frames) if isinstance(layout, str) else list(layout)
    for lay in layouts if layouts else [layout]:
        if not isinstance(lay, str) or lay not in LAYOUTS:
            raise Yfv2Error("resize_frames: layout must be one of %s, got %r" % (", ".join(LAYOUTS), lay))
    if not frames:
        raise Yfv2Error("resize_frames: no frames")
    if len(layouts) != len(frames):
        raise Yfv2Error("resize_frames: %d layouts for %d frames" % (len(layouts), len(frames)))
    checked = [_check_frame(f, lay, i) for i, (f, lay) in enumerate(zip(frames, layouts))]
    if device is None:
        cuda = [t.device for f in checked for t in (f if isinstance(f, (tuple, list)) else (f,))
                if isinstance(t, torch.Tensor) and t.is_cuda]
        device = cuda[0] if cuda else torch.device("cuda", torch.cuda.current_device())
    device = torch.device(device)
    if device.type != "cuda":
        raise Yfv2Error("resize_frames: runs on CUDA devices only (no CPU fallback)")
    N = len(frames)
    if out is None:
        out = torch.empty((N, 3, H, W), dtype=torch.uint8, device=device)
    elif tuple(out.shape) != (N, 3, H, W) or out.dtype != torch.uint8 or not out.is_contiguous() or out.device != device:
        raise Yfv2Error("resize_frames: out must be a contiguous uint8 tensor of shape %s on %s" % ((N, 3, H, W), device))
    i = 0
    while i < N:
        kind, j = _KIND[layouts[i]], i + 1
        while j < N and _KIND[layouts[j]] == kind:
            j += 1
        if kind == "bgr":
            resize_bgr(checked[i:j], W, H, device, out[i:j])
        elif kind == "yuv420":
            resize_yuv420(checked[i:j], W, H, layouts[i:j], device, out[i:j])
        else:
            _resize_layout_run(checked[i:j], layouts[i:j], W, H, device, out[i:j])
        i = j
    return out


def crop_frame(frame, layout, x0, y0, w, h):
    """The w x h window at (x0, y0) of a frame, in the form resize_frames takes for `layout`, as a view (nothing is copied):
    resize_frames of the crop gives the bytes of cv2.resize(cv2.cvtColor(frame, COLOR_<LAYOUT>2BGR)[y0:y0+h, x0:x0+w]).  HWC
    layouts and grey are sliced in place, "rgb_chw" as [3, h, w].  A 4:2:0 frame (a single [h*3/2, w] buffer or its planes)
    becomes a tuple of cropped planes, (y, uv) for NV12 / NV21 and (y, u, v) for I420 / YV12; x0, y0, w, h must then be even, so
    that the 2x2 chroma blocks of the crop are those of the frame.  Packed 4:2:2 needs even x0 and w (whole macropixels)."""
    if layout not in LAYOUTS:
        raise Yfv2Error("crop_frame: layout must be one of %s, got %r" % (", ".join(LAYOUTS), layout))
    f = _check_frame(frame, layout, 0)
    fh, fw = frame_size(f, layout)
    x0, y0, w, h = int(x0), int(y0), int(w), int(h)
    if w < 1 or h < 1 or x0 < 0 or y0 < 0 or x0 + w > fw or y0 + h > fh:
        raise Yfv2Error("crop_frame: window (x0 %d, y0 %d, %dx%d) is not inside the %dx%d frame" % (x0, y0, w, h, fw, fh))
    if layout in YUV420_LAYOUTS and (x0 | y0 | w | h) & 1:
        raise Yfv2Error("crop_frame: %s crops need even x0, y0, w and h (2x2 chroma blocks), got (x0 %d, y0 %d, %dx%d)"
                        % (layout, x0, y0, w, h))
    if layout in YUV422_LAYOUTS and (x0 | w) & 1:
        raise Yfv2Error("crop_frame: %s crops need even x0 and w (two pixels per macropixel), got x0 %d, w %d" % (layout, x0, w))
    if layout in YUV420_LAYOUTS:
        y, u, v = _yuv420_planes(f, layout, 0)
        cy = slice(y0 // 2, (y0 + h) // 2)
        if layout in ("nv12", "nv21"):
            return y[y0:y0 + h, x0:x0 + w], u[cy, x0:x0 + w]
        cx = slice(x0 // 2, (x0 + w) // 2)
        return y[y0:y0 + h, x0:x0 + w], u[cy, cx], v[cy, cx]
    if layout == "rgb_chw":
        return f[:, y0:y0 + h, x0:x0 + w]
    return f[y0:y0 + h, x0:x0 + w]


def debug_pw_tc(x, w):
    """out[n][p] = sum_k w[n][k] * x[k][p] on the 3xTF32 tensor-core engine (test hook)."""
    _require_cuda(x, "x"); _require_cuda(w, "w")
    K, P = x.shape
    N = w.shape[0]
    out = torch.empty((N, P), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        _check(lib().yfv2_debug_pw_tc(ctypes.c_void_p(x.contiguous().data_ptr()), ctypes.c_void_p(w.contiguous().data_ptr()),
                                      ctypes.c_void_p(out.data_ptr()), None, K, N, P, _stream(x.device)),
               "debug_pw_tc")
    return out


def loss_geometry(preds, cfg):
    """(N, H, W, A, C) of the six head tensors, checked against each other and against cfg.  The kernel takes A, C and the
    input size from the tensors while the reference takes anchor_num, classes and width / height from cfg (utils/loss.py:56,81,
    148,198), so a cfg that disagrees with the tensors would silently select other anchors or another CE divisor: ValueError."""
    if len(preds) != 6:
        raise ValueError("compute_loss: expected the six head tensors, got %d" % len(preds))
    N, _, h, w = preds[0].shape
    A, C = preds[1].shape[1], preds[2].shape[1]
    H, W = h * 16, w * 16
    want = [(N, 4 * A, h, w), (N, A, h, w), (N, C, h, w), (N, 4 * A, h // 2, w // 2), (N, A, h // 2, w // 2),
            (N, C, h // 2, w // 2)]
    got = [tuple(p.shape) for p in preds]
    if got != want or h % 2 or w % 2:
        raise ValueError("compute_loss: head tensor shapes %s are not those of one %dx%d input with %d anchors and %d classes"
                         % (got, H, W, A, C))
    bad = []
    if int(cfg["anchor_num"]) != A:
        bad.append("anchor_num %s (the heads have %d anchors)" % (cfg["anchor_num"], A))
    if int(cfg["classes"]) != C:
        bad.append("classes %s (the heads have %d)" % (cfg["classes"], C))
    if float(cfg["width"]) != W or float(cfg["height"]) != H:
        bad.append("width x height %s x %s (the heads are those of a %d x %d input)" % (cfg["width"], cfg["height"], W, H))
    if len(cfg["anchors"]) != 4 * A:
        bad.append("%d anchor values (two levels of %d anchors need %d)" % (len(cfg["anchors"]), A, 4 * A))
    if bad:
        raise ValueError("compute_loss: cfg disagrees with the head tensors: " + "; ".join(bad))
    return N, H, W, A, C


def compute_loss(preds, targets, cfg, want_grads=True, return_workspace=False):
    """utils.loss.compute_loss on the device.  Returns (losses[4] CUDA tensor, dpreds 6-tuple or None[, workspace])."""
    for p in preds:
        _require_cuda(p, "preds")
    N, H, W, A, C = loss_geometry(preds, cfg)
    preds = [p.detach().contiguous().float() for p in preds]
    dev = preds[0].device
    targets = targets.detach().to(dev).float().contiguous().reshape(-1, 6)
    nt = targets.shape[0]
    nb = ctypes.c_size_t()
    _check(lib().yfv2_loss_workspace_bytes(N, H, W, A, C, nt, ctypes.byref(nb)), "loss_workspace_bytes")
    ws = torch.empty(nb.value, dtype=torch.uint8, device=dev)
    losses = torch.empty(4, dtype=torch.float32, device=dev)
    dpreds = [torch.empty_like(p) for p in preds] if want_grads else None
    with torch.cuda.device(dev):
        _check(lib().yfv2_compute_loss(_ptr_array(preds), ctypes.c_void_p(targets.data_ptr()) if nt else None, nt, N, H, W, A, C,
                                       anchors_array(cfg), ctypes.c_void_p(losses.data_ptr()),
                                       _ptr_array(dpreds) if want_grads else None, ctypes.c_void_p(ws.data_ptr()), _stream(dev)),
               "compute_loss")
    out = (losses, tuple(dpreds) if want_grads else None)
    return out + ((ws, (N, H, W, A, nt)),) if return_workspace else out


def read_targets(ws_info, level):
    """Matched rows of one level after compute_loss(..., return_workspace=True): (idx[4,m], tbox[m,4], anch[m,2], tcls[m])."""
    ws, (N, H, W, A, nt) = ws_info
    cap = 5 * A * max(nt, 1)
    dev = ws.device
    idx = torch.zeros((4, cap), dtype=torch.int32, device=dev)
    tbox = torch.zeros((cap, 4), dtype=torch.float32, device=dev)
    anch = torch.zeros((cap, 2), dtype=torch.float64, device=dev)
    tcls = torch.zeros((cap,), dtype=torch.int32, device=dev)
    cnt = ctypes.c_int()
    with torch.cuda.device(dev):
        _check(lib().yfv2_loss_read_targets(ctypes.c_void_p(ws.data_ptr()), level, N, H, W, A, nt, ctypes.byref(cnt),
                                            ctypes.c_void_p(idx.data_ptr()), ctypes.c_void_p(tbox.data_ptr()),
                                            ctypes.c_void_p(anch.data_ptr()), ctypes.c_void_p(tcls.data_ptr()), _stream(dev)),
               "loss_read_targets")
    m = cnt.value
    return idx[:, :m], tbox[:m], anch[:m], tcls[:m]


def op(name, tensors_and_ints, device):
    """Calls yfv2_op_<name>: tensors become data pointers (None -> NULL), ints pass through, the stream is appended."""
    args = []
    for a in tensors_and_ints:
        if a is None:
            args.append(None)
        elif isinstance(a, torch.Tensor):
            args.append(ctypes.c_void_p(a.data_ptr()))
        else:
            args.append(int(a))
    with torch.cuda.device(device):
        _check(getattr(lib(), "yfv2_op_" + name)(*args, _stream(device)), "op_" + name)


def export_heads(preds):
    """Detector(..., export_onnx=True) output: two channel-last [N,h,w,5A+C] tensors (sigmoid / sigmoid / softmax)."""
    preds = [p.detach().contiguous().float() for p in preds]
    N, _, h, w = preds[0].shape
    A, C = preds[1].shape[1], preds[2].shape[1]
    dev = preds[0].device
    o2 = torch.empty((N, h, w, 5 * A + C), dtype=torch.float32, device=dev)
    o3 = torch.empty((N, preds[3].shape[2], preds[3].shape[3], 5 * A + C), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _check(lib().yfv2_export_heads(_ptr_array(preds), N, h * 16, w * 16, A, C, ctypes.c_void_p(o2.data_ptr()),
                                       ctypes.c_void_p(o3.data_ptr()), _stream(dev)), "export_heads")
    return o2, o3


NCNN_ANCHORS = (12.64, 19.39, 37.88, 51.48, 55.71, 138.31, 126.91, 78.23, 131.57, 214.55, 279.92, 258.87)   # sample/ncnn/src/yolo-fastestv2.cpp:34-35


def ncnn_post(out2, out3, anchor_num, thresh=0.3, nms_thresh=0.25, src_size=None, anchors=NCNN_ANCHORS, max_out=None):
    """The deploy post-process of the reference's ncnn sample (yoloFastestv2::detection after the forward: predHandle + nmsHandle,
    sample/ncnn/src/yolo-fastestv2.cpp:78-183) on the export_onnx tensors `out2` [N,h,w,5A+C], `out3` (export_heads above).
    src_size = (cols, rows) of the source image (default: the network input size, scale 1).  Returns a list of N tuples
    (boxes int32 [n,4], scores float32 [n], cates int32 [n]) on the CPU, descending score, like the sample's dstBoxes."""
    if not (out2.is_cuda and out3.is_cuda):
        raise RuntimeError("yfv2: ncnn_post needs CUDA tensors (there is no CPU fallback)")
    out2 = out2.detach().contiguous().float(); out3 = out3.detach().contiguous().float()
    N, h, w, ch = out2.shape
    A = int(anchor_num)
    C = ch - 5 * A
    H, W = h * 16, w * 16
    M = A * (h * w + out3.shape[1] * out3.shape[2])
    max_out = M if max_out is None else int(max_out)
    sw, sh = (W, H) if src_size is None else src_size
    import numpy as np
    scale_w = float(np.float32(sw) / np.float32(W)); scale_h = float(np.float32(sh) / np.float32(H))        # :189-190, float division
    dev = out2.device
    boxes = torch.empty((N, max_out, 4), dtype=torch.int32, device=dev)
    scores = torch.empty((N, max_out), dtype=torch.float32, device=dev)
    cates = torch.empty((N, max_out), dtype=torch.int32, device=dev)
    counts = torch.empty((N,), dtype=torch.int32, device=dev)
    if len(anchors) < 4 * A:
        raise Yfv2Error("ncnn_post: %d anchor values given, 2 levels x %d anchors x (w, h) needed" % (len(anchors), A))
    if C <= 0:
        raise Yfv2Error("ncnn_post: tensors with %d channels cannot hold %d anchors" % (ch, A))
    anc = (ctypes.c_float * (4 * A))(*[float(a) for a in anchors][:4 * A])
    with torch.cuda.device(dev):
        _check(lib().yfv2_ncnn_post(ctypes.c_void_p(out2.data_ptr()), ctypes.c_void_p(out3.data_ptr()), N, H, W, A, C, anc,
                                    ctypes.c_float(thresh), ctypes.c_float(nms_thresh), ctypes.c_float(scale_w), ctypes.c_float(scale_h),
                                    max_out, ctypes.c_void_p(boxes.data_ptr()), ctypes.c_void_p(scores.data_ptr()),
                                    ctypes.c_void_p(cates.data_ptr()), ctypes.c_void_p(counts.data_ptr()), _stream(dev)), "ncnn_post")
    cnt = counts.cpu().tolist()
    b, s, c = boxes.cpu(), scores.cpu(), cates.cpu()
    return [(b[i, :min(cnt[i], max_out)].numpy(), s[i, :min(cnt[i], max_out)].numpy(), c[i, :min(cnt[i], max_out)].numpy()) for i in range(N)]

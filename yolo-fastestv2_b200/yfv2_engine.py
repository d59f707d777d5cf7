"""ctypes binding of libyfv2.so (include/yfv2.h) plus the small amount of host bookkeeping the Python
mirror modules share: plan cache, weight packing, output allocation.  PyTorch is used for device
memory and streams only; every device computation is a kernel inside libyfv2.so.

There is NO CPU fallback: if the library is missing or the tensors are not on a CUDA device the calls
raise.
"""
import collections
import ctypes
import os
import threading

import numpy as np
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


class _EncFrame(ctypes.Union):
    _fields_ = [("bgr", Frame), ("strided", StridedFrame), ("yuv420", Yuv420Frame), ("yuv422", Yuv422Frame)]


class JpegEncSrc(ctypes.Structure):
    """yfv2_jpeg_enc_src: one output of yfv2_jpeg_encode: a frame, its region and cv2.imencode's params."""
    _fields_ = [("kind", ctypes.c_int), ("x0", ctypes.c_int), ("y0", ctypes.c_int), ("w", ctypes.c_int), ("h", ctypes.c_int),
                ("f", _EncFrame), ("params", ctypes.POINTER(ctypes.c_int)), ("nparams", ctypes.c_int)]


class TrainerOp(ctypes.Structure):
    """yfv2_trainer_op: one op of the native trainer's program (test hook)."""
    _fields_ = [(f, ctypes.c_int) for f in ("kind", "a", "b", "y", "pw", "pg", "pb", "pbias", "bn", "relu", "ks", "stride", "M")] + \
               [("aux", ctypes.c_longlong)]


class TrainerBwdOp(ctypes.Structure):
    """yfv2_trainer_bwd_op: one op whose backward runs under the trainer's current mode, and what it writes (test hook)."""
    _fields_ = [(f, ctypes.c_int) for f in ("op", "da", "db", "dw", "dbias", "dgamma", "dbeta", "bn_eval")]


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


def trainer_backward_plan(handle):
    """The ops whose backward runs under a yfv2_trainer handle's current mode, in backward order, as dicts (host only; test hook)."""
    L, n = lib(), ctypes.c_int()
    _check(L.yfv2_trainer_debug_backward(handle, None, 0, ctypes.byref(n)), "trainer_debug_backward")
    recs = (TrainerBwdOp * n.value)()
    _check(L.yfv2_trainer_debug_backward(handle, recs, n.value, ctypes.byref(n)), "trainer_debug_backward")
    return [{f: getattr(r, f) for f, _ in r._fields_} for r in recs]


def trainer_mode(trainable=None, bn_eval=None):
    """(trainable, bn_eval) as tuples of bools, None for the default (all trainable / all train mode); a flag list of the wrong
    length raises (225 parameters, 73 BatchNorm layers)."""
    trainable = None if trainable is None else tuple(bool(v) for v in trainable)
    bn_eval = None if bn_eval is None else tuple(bool(v) for v in bn_eval)
    if trainable is not None and len(trainable) != 225:
        raise Yfv2Error("trainer mode: %d trainable flags, expected 225 (one per parameter)" % len(trainable))
    if bn_eval is not None and len(bn_eval) != 73:
        raise Yfv2Error("trainer mode: %d bn_eval flags, expected 73 (one per BatchNorm layer)" % len(bn_eval))
    return (None if trainable is None or all(trainable) else trainable,
            None if bn_eval is None or not any(bn_eval) else bn_eval)


def trainer_set_mode(handle, trainable, bn_eval):
    """yfv2_trainer_set_mode on a handle (host only); arguments as trainer_mode returns them."""
    arr = lambda v: None if v is None else (ctypes.c_ubyte * len(v))(*v)
    _check(lib().yfv2_trainer_set_mode(handle, arr(trainable), arr(bn_eval)), "trainer_set_mode")


class LaunchRecord(ctypes.Structure):
    """yfv2_launch: one kernel launch of a forward, as the forward chooses it (test hook)."""
    _fields_ = [("kernel", ctypes.c_char * 32), ("first", ctypes.c_int), ("last", ctypes.c_int), ("smem", ctypes.c_longlong),
                ("grid", ctypes.c_int * 3)] + [(f, ctypes.c_int) for f in ("persistent", "items", "R", "bands", "G", "window_stride")]


def plan_launches(handle, workspace=None, is_u8=False, sms=0):
    """The kernel launches of a whole forward of a yfv2_plan handle, in order, as dicts (yfv2_plan_debug_launches; host only).
    workspace None: a 16-byte-aligned workspace; sms 0: this device's SM count."""
    L, n = lib(), ctypes.c_int()
    ws = ctypes.c_void_p(workspace)
    _check(L.yfv2_plan_debug_launches(handle, ws, int(is_u8), sms, None, 0, ctypes.byref(n)), "plan_debug_launches")
    recs = (LaunchRecord * n.value)()
    _check(L.yfv2_plan_debug_launches(handle, ws, int(is_u8), sms, recs, n.value, ctypes.byref(n)), "plan_debug_launches")
    out = []
    for r in recs:
        d = {f: getattr(r, f) for f, _ in r._fields_}
        d["kernel"], d["grid"], d["persistent"] = r.kernel.decode(), tuple(r.grid), bool(r.persistent)
        out.append(d)
    return out


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


class TrackParams(ctypes.Structure):
    """yfv2_track_params: the tracker's thresholds and the frames a lost track survives."""
    _fields_ = [("high_thresh", ctypes.c_double), ("low_thresh", ctypes.c_double), ("new_thresh", ctypes.c_double),
                ("match_thresh", ctypes.c_double), ("max_age", ctypes.c_int)]


class TrackRecord(ctypes.Structure):
    """yfv2_track: one track's state as yfv2_track_debug_read copies it."""
    _fields_ = [("mean", ctypes.c_double * 8), ("cov", ctypes.c_double * 12), ("score", ctypes.c_double), ("cls", ctypes.c_double),
                ("id", ctypes.c_int), ("state", ctypes.c_int), ("confirmed", ctypes.c_int), ("start_frame", ctypes.c_int),
                ("end_frame", ctypes.c_int), ("det_row", ctypes.c_int)]


TRACK_TRACKED, TRACK_LOST = 1, 2                     # yfv2_track.state
TRACK_MAX_CAPACITY, TRACK_MAX_ROWS, TRACK_MAX_BATCH = 1024, 2048, 4096


class AugParams(ctypes.Structure):
    """yfv2_aug_params: one image's contrast (alpha, beta) and random_resize size (rw, rh)."""
    _fields_ = [("alpha", ctypes.c_float), ("beta", ctypes.c_float), ("rw", ctypes.c_int), ("rh", ctypes.c_int)]


AUG_CONTRAST, AUG_RESIZE, AUG_HSV = 1, 2, 4          # yfv2_aug_batch flags (include/yfv2.h)
AUG_BLUR = 8                                         # yfv2_aug_batch_blur adds motion_blur


class AugBlur(ctypes.Structure):
    """yfv2_aug_blur: one image's motion_blur kernel (ksize 0: the image drew no blur)."""
    _fields_ = [("ksize", ctypes.c_int), ("taps", ctypes.c_float * 9)]


class JpegInfo(ctypes.Structure):
    """yfv2_jpeg_info: what yfv2_jpeg_parse found in one file."""
    _fields_ = [("status", ctypes.c_int), ("w", ctypes.c_int), ("h", ctypes.c_int), ("components", ctypes.c_int),
                ("h_samp", ctypes.c_int), ("v_samp", ctypes.c_int), ("orientation", ctypes.c_int), ("restart_interval", ctypes.c_int),
                ("segments", ctypes.c_int), ("scans", ctypes.c_int), ("frame_offset", ctypes.c_longlong), ("reason", ctypes.c_char * 96)]


JPEG_ENTROPY, JPEG_IDCT, JPEG_COLOR, JPEG_ALL = 1, 2, 4, 7     # yfv2_jpeg_decode phases
JPEG_PROGRESSIVE = 1                                          # yfv2_jpeg_parse_ex flags


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
    "yfv2_track_state_bytes": (ctypes.c_int, [ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_size_t)]),
    "yfv2_track_reset": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_int), ctypes.c_int,
                                        ctypes.c_void_p]),
    "yfv2_track_update": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_int), ctypes.c_int,
                                         ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(TrackParams), ctypes.c_void_p,
                                         ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "yfv2_track_debug_read": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_int),
                                             ctypes.POINTER(ctypes.c_int), ctypes.POINTER(TrackRecord), ctypes.POINTER(ctypes.c_int),
                                             ctypes.c_void_p]),
    "yfv2_batch_statistics": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                             ctypes.c_int, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p]),
    "yfv2_aug_contrast_brightness": (ctypes.c_int, [ctypes.c_void_p] * 4 + [ctypes.c_int, ctypes.c_longlong, ctypes.c_void_p]),
    "yfv2_aug_batch": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                      ctypes.POINTER(AugParams), ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]),
    "yfv2_aug_blur_workspace_bytes": (ctypes.c_int, [ctypes.c_int] * 3 + [ctypes.POINTER(ctypes.c_size_t)]),
    "yfv2_aug_batch_blur": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                           ctypes.POINTER(AugParams), ctypes.c_void_p, ctypes.POINTER(AugBlur), ctypes.c_int,
                                           ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "yfv2_debug_bgr2hsv": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p]),
    "yfv2_debug_hsv2bgr": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int, ctypes.c_void_p]),
    "yfv2_jpeg_encode_plan": (ctypes.c_int, [ctypes.POINTER(JpegEncSrc), ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t,
                                             ctypes.POINTER(ctypes.c_size_t), ctypes.POINTER(ctypes.c_size_t),
                                             ctypes.POINTER(ctypes.c_longlong), ctypes.POINTER(ctypes.c_size_t)]),
    "yfv2_jpeg_encode": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t,
                                        ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]),
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
    "yfv2_op_bn_eval_fwd": (ctypes.c_int, [ctypes.c_void_p] * 8 + [ctypes.c_int] * 4 + [ctypes.c_void_p]),
    "yfv2_op_bn_eval_bwd": (ctypes.c_int, [ctypes.c_void_p] * 10 + [ctypes.c_int] * 4 + [ctypes.c_void_p]),
    "yfv2_op_maxpool_fwd": (ctypes.c_int, [ctypes.c_void_p] * 3 + [ctypes.c_int] * 3 + [ctypes.c_void_p]),
    "yfv2_op_maxpool_bwd": (ctypes.c_int, [ctypes.c_void_p] * 3 + [ctypes.c_int] * 3 + [ctypes.c_void_p]),
    "yfv2_op_upsample2_fwd": (ctypes.c_int, [ctypes.c_void_p] * 2 + [ctypes.c_int] * 3 + [ctypes.c_void_p]),
    "yfv2_op_upsample2_bwd": (ctypes.c_int, [ctypes.c_void_p] * 2 + [ctypes.c_int] * 3 + [ctypes.c_void_p]),
    "yfv2_trainer_create": (ctypes.c_int, [_c_void_pp] + [ctypes.c_int] * 6),
    "yfv2_trainer_destroy": (None, [ctypes.c_void_p]),
    "yfv2_trainer_workspace_bytes": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_size_t)]),
    "yfv2_trainer_grad_floats": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_longlong)]),
    "yfv2_trainer_param_offset": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_longlong), ctypes.POINTER(ctypes.c_longlong)]),
    "yfv2_trainer_set_mode": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "yfv2_trainer_debug_backward": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_int)]),
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
    "yfv2_plan_debug_launches": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                                ctypes.c_int, ctypes.POINTER(ctypes.c_int)]),
    "yfv2_jpeg_parse": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t,
                                       ctypes.POINTER(ctypes.c_size_t), ctypes.POINTER(ctypes.c_size_t), ctypes.POINTER(ctypes.c_size_t)]),
    "yfv2_jpeg_parse_ex": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                          ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t), ctypes.POINTER(ctypes.c_size_t),
                                          ctypes.POINTER(ctypes.c_size_t)]),
    "yfv2_jpeg_decode": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p,
                                        ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p]),
    "yfv2_jpeg_decode_resize": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t,
                                               ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                               ctypes.c_size_t, ctypes.c_void_p]),
    "yfv2_anchor_kmeans_step": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int] +
                                [ctypes.c_void_p] * 7),
    "yfv2_anchor_avg_iou": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                           ctypes.c_void_p]),
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
        self.mode = (None, None)              # (trainable, bn_eval) tuples of bools; None: the default (all trainable, all train)
        self._read_layout()
        self.generation = 0                  # bumped by every forward: a backward must see the generation of its own forward
        # persistent buffers: the C side replays its two programs as CUDA graphs while every pointer stays the same
        self.x_static = torch.empty((N, 3, H, W), dtype=torch.float32, device=self.device)
        self.preds_static = self.alloc_preds()
        self.dpreds_static = [torch.empty_like(p) for p in self.preds_static]
        self.flat_static = torch.empty(self.grad_floats, dtype=torch.float32, device=self.device)

    def _read_layout(self):
        """grad_floats and param_offsets ((offset, numel) per parameter, offset -1 when frozen) of the current mode."""
        L = lib()
        n = ctypes.c_longlong()
        _check(L.yfv2_trainer_grad_floats(self._h, ctypes.byref(n)), "trainer_grad_floats")
        self.grad_floats = n.value
        self.param_offsets = []
        off, num = ctypes.c_longlong(), ctypes.c_longlong()
        for i in range(225):
            _check(L.yfv2_trainer_param_offset(self._h, i, ctypes.byref(off), ctypes.byref(num)), "trainer_param_offset")
            self.param_offsets.append((off.value, num.value))

    def set_mode(self, trainable=None, bn_eval=None):
        """Fine-tuning mode from the next forward(): trainable = 225 flags (p.requires_grad in model.parameters() order), bn_eval =
        73 flags (BatchNorm module not .training, in module order); None: all trainable / all train mode.  Cheap when unchanged."""
        mode = trainer_mode(trainable, bn_eval)
        if mode == self.mode:
            return
        trainer_set_mode(self._h, *mode)
        self.mode = mode
        self._read_layout()
        if self.flat_static.numel() != self.grad_floats:
            self.flat_static = torch.empty(self.grad_floats, dtype=torch.float32, device=self.device)

    def backward_plan(self):
        """trainer_backward_plan of the current mode (host only)."""
        return trainer_backward_plan(self._h)

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

    def launches(self, is_u8=False, sms=0):
        """The kernel launches of a forward on this plan's workspace (plan_launches; host only)."""
        return plan_launches(self._h, self.workspace.data_ptr(), is_u8, sms)

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
        """Whole step from pinned host uint8 images to pinned host detections (asynchronous).  x_host: uint8 [N,3,H,W], out_host:
        float32 [N,max_det,6], counts_host: int32 [N], contiguous CPU tensors (pinned, so that the copies overlap); anchors: the
        4*A doubles of anchors_array.  The plan must have been built with detect_max_det >= max_det."""
        for t, name, dtype, shape in ((x_host, "x_host", torch.uint8, (self.N, 3, self.H, self.W)),
                                      (out_host, "out_host", torch.float32, (self.N, max_det, 6)),
                                      (counts_host, "counts_host", torch.int32, (self.N,))):
            if (not isinstance(t, torch.Tensor) or t.device.type != "cpu" or t.dtype != dtype or tuple(t.shape) != shape
                    or not t.is_contiguous()):
                got = "%s %s on %s" % (t.dtype, tuple(t.shape), t.device) if isinstance(t, torch.Tensor) else type(t).__name__
                raise Yfv2Error("detect_u8_host: %s must be a contiguous host tensor %s %s, got %s" % (name, dtype, shape, got))
        if not isinstance(anchors, ctypes.Array) or anchors._type_ is not ctypes.c_double or len(anchors) < 4 * self.A:
            raise Yfv2Error("detect_u8_host: anchors must be %d doubles (anchors_array)" % (4 * self.A))
        need = lib().yfv2_detect_workspace_bytes(self._h, max_det)
        if max_det > 0 and self.workspace.numel() < need:
            raise Yfv2Error("detect_u8_host: max_det=%d needs a %d-byte workspace, the plan has %d (build it with detect_max_det >= %d)"
                            % (max_det, need, self.workspace.numel(), max_det))
        with torch.cuda.device(self.device):
            _check(lib().yfv2_detect_u8_host(self._h, ctypes.c_void_p(x_host.data_ptr()), ctypes.c_void_p(self.packed.data_ptr()),
                                             anchors, ctypes.c_float(conf_thres), ctypes.c_double(iou_thres), max_det,
                                             ctypes.c_void_p(out_host.data_ptr()), ctypes.c_void_p(counts_host.data_ptr()),
                                             ctypes.c_void_p(self.workspace.data_ptr()), _stream(self.device)), "detect_u8_host")


def _expect_shapes(what, tensors, names, shapes):
    """Raises Yfv2Error naming the first tensor that is not a CUDA tensor on tensors[0]'s device with the expected shape.  The
    kernels take every extent from a few of these tensors and read the others blindly, so a mismatch would be an out-of-bounds
    device read."""
    dev = tensors[0].device if isinstance(tensors[0], torch.Tensor) else None
    for t, name, want in zip(tensors, names, shapes):
        _require_cuda(t, "%s: %s" % (what, name))
        if t.device != dev:
            raise Yfv2Error("%s: %s is on %s, expected %s like %s" % (what, name, t.device, dev, names[0]))
        if tuple(t.shape) != tuple(want):
            raise Yfv2Error("%s: %s has shape %s, expected %s" % (what, name, tuple(t.shape), tuple(want)))


def head_geometry(what, preds):
    """(N, h, w, A, C) of the six head tensors (reg, obj, cls of the stride-16 level, then of the stride-32 level), checked
    against each other: preds[0] gives N, h, w, preds[1] A and preds[2] C; every tensor must match them, and the stride-32 maps
    are (h/2, w/2) of an input whose sides are multiples of 32."""
    if len(preds) != 6:
        raise Yfv2Error("%s: expected preds to be the 6-tuple (reg,obj,cls) x 2 levels, got %d tensors" % (what, len(preds)))
    for i, p in enumerate(preds):
        _require_cuda(p, "%s: preds[%d]" % (what, i))
        if p.dim() != 4:
            raise Yfv2Error("%s: preds[%d] has shape %s, expected [N, channels, rows, columns]" % (what, i, tuple(p.shape)))
    N, _, h, w = preds[0].shape
    A, C = preds[1].shape[1], preds[2].shape[1]
    if h % 2 or w % 2 or h == 0 or w == 0:
        raise Yfv2Error("%s: preds[0] has shape %s: %dx%d maps are not those of an input whose sides are multiples of 32"
                        % (what, tuple(preds[0].shape), h, w))
    want = [(N, 4 * A, h, w), (N, A, h, w), (N, C, h, w), (N, 4 * A, h // 2, w // 2), (N, A, h // 2, w // 2), (N, C, h // 2, w // 2)]
    _expect_shapes(what, preds, ["preds[%d]" % i for i in range(6)], want)
    return N, h, w, A, C


def decode(preds, cfg):
    """handel_preds on the device: returns [N, M, 5+C] fp32 CUDA tensor."""
    N, h, w, A, C = head_geometry("decode", preds)
    preds = [p.detach().contiguous().float() for p in preds]
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
    N, h, w, A, C = head_geometry("decode_nms", preds)
    preds = [p.detach().contiguous().float() for p in preds]
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


class Tracker:
    """A multi-stream tracker (yfv2_track_*, include/yfv2.h): ByteTrack's association in three stages and its track lifecycle with
    a constant-velocity Kalman filter, for `streams` streams (cameras) of at most `capacity` tracks each.  It owns the device state
    tensor; every stream starts reset (no tracks, frame 0, next id 1).  Class-agnostic: a track takes the class of its latest
    detection."""

    def __init__(self, device, streams, capacity, high_thresh=0.5, low_thresh=0.1, new_thresh=0.6, match_thresh=0.8, max_age=30):
        self.device = torch.device(device)
        self.S, self.K = int(streams), int(capacity)
        self.params = TrackParams(float(high_thresh), float(low_thresh), float(new_thresh), float(match_thresh), int(max_age))
        nb = ctypes.c_size_t()
        _check(lib().yfv2_track_state_bytes(self.S, self.K, ctypes.byref(nb)), "Tracker")
        self.state = torch.zeros((nb.value,), dtype=torch.uint8, device=self.device)
        self.reset()

    @property
    def low_thresh(self):
        return self.params.low_thresh

    def _streams(self, streams, B):
        idx = list(range(B)) if streams is None else [int(s) for s in streams]
        return idx, (ctypes.c_int * max(len(idx), 1))(*idx)

    def reset(self, streams=None):
        """Clears the given streams (all by default): no tracks, frame 0, next id 1."""
        idx, arr = self._streams(streams, self.S)
        with torch.cuda.device(self.device):
            _check(lib().yfv2_track_reset(ctypes.c_void_p(self.state.data_ptr()), self.S, self.K, arr, len(idx), _stream(self.device)),
                   "Tracker.reset")

    def update(self, dets, counts, streams=None):
        """One frame for each of B distinct streams (streams: B stream indices; None: 0..B-1), in one launch without a host
        synchronisation.  dets: CUDA float64 [B, M, 6] rows (x1, y1, x2, y2, conf, cls) in frame pixels, counts int32 [B] (what
        merge_regions returns).  Returns CUDA tensors (out float64 [B, capacity, 8]: the confirmed tracked tracks in ascending id,
        (x1, y1, x2, y2, score, cls, track_id, det_row), zeros past the count; counts int32 [B]; dropped int32 [B]: births refused
        for want of capacity)."""
        _require_cuda(dets, "dets")
        _require_cuda(counts, "counts")
        if dets.dim() != 3 or dets.shape[2] != 6 or dets.dtype != torch.float64:
            raise Yfv2Error("Tracker.update: dets must be float64 [B, M, 6], got %s %s" % (dets.dtype, tuple(dets.shape)))
        B, M = dets.shape[0], dets.shape[1]
        if counts.dtype != torch.int32 or tuple(counts.shape) != (B,):
            raise Yfv2Error("Tracker.update: counts must be int32 [%d], got %s %s" % (B, counts.dtype, tuple(counts.shape)))
        idx, arr = self._streams(streams, B)
        if len(idx) != B:
            raise Yfv2Error("Tracker.update: %d streams for %d row blocks" % (len(idx), B))
        dets, counts = dets.contiguous(), counts.contiguous()
        out = torch.empty((B, self.K, 8), dtype=torch.float64, device=self.device)
        out_counts = torch.empty((B,), dtype=torch.int32, device=self.device)
        dropped = torch.empty((B,), dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            _check(lib().yfv2_track_update(ctypes.c_void_p(self.state.data_ptr()), self.S, self.K, arr, B, ctypes.c_void_p(dets.data_ptr()),
                                           ctypes.c_void_p(counts.data_ptr()), M, ctypes.byref(self.params),
                                           ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(out_counts.data_ptr()),
                                           ctypes.c_void_p(dropped.data_ptr()), _stream(self.device)), "Tracker.update")
        return out, out_counts, dropped

    def tracks(self, stream):
        """Stream `stream`'s state on the host (test hook; synchronises): {"frame", "next_id", "tracks"}, the live tracks in
        ascending id as dicts (id, cls, state, confirmed, start_frame, end_frame, score, det_row, mean [8], cov [12])."""
        recs = (TrackRecord * self.K)()
        frame, next_id, n = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        with torch.cuda.device(self.device):
            _check(lib().yfv2_track_debug_read(ctypes.c_void_p(self.state.data_ptr()), self.S, self.K, int(stream), ctypes.byref(frame),
                                               ctypes.byref(next_id), recs, ctypes.byref(n), _stream(self.device)), "Tracker.tracks")
        keys = ("id", "cls", "state", "confirmed", "start_frame", "end_frame", "score", "det_row")
        tracks = [dict({k: getattr(r, k) for k in keys}, mean=list(r.mean), cov=list(r.cov)) for r in recs[:n.value]]
        return {"frame": frame.value, "next_id": next_id.value, "tracks": tracks}


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


def hsv_luts(r):
    """augment_hsv's LUTs (utils/datasets.py:44-47) for gains r [N, 3] (hue, saturation, value): uint8 [N, 3, 256], built with
    the reference's arithmetic (int16 x times the float64 gain, floor-mod 180 / clip to 0..255, truncation to uint8)."""
    import numpy as np
    r = np.asarray(r, dtype=np.float64).reshape(-1, 3)
    x = np.arange(0, 256, dtype=np.int16)
    out = np.empty((r.shape[0], 3, 256), np.uint8)
    for n, g in enumerate(r):
        out[n, 0] = ((x * g[0]) % 180).astype(np.uint8)
        out[n, 1] = np.clip(x * g[1], 0, 255).astype(np.uint8)
        out[n, 2] = np.clip(x * g[2], 0, 255).astype(np.uint8)
    return out


def motion_blur_taps(degree, angle):
    """motion_blur's kernel (utils/datasets.py:25-29) as filter2D applies it: fp32 [degree, degree], degree 2 or 3.

    cv2.warpAffine(np.diag(np.ones(degree)), cv2.getRotationMatrix2D((degree/2, degree/2), angle, 1), (degree, degree)) / degree
    restated without cv2: the rotation with libm cos / sin in fp64, inverted as warpAffine inverts it, each destination pixel's
    source position in warpAffine's fixed point (cvRound of the 1024-scaled terms, + 16, >> 5: 1/32-pixel steps), fp32 bilinear
    weights, pixels outside the 0/1 diagonal image read as 0, the fp64 weighted sum; then / degree in fp64 and rounded to fp32."""
    import math
    import numpy as np
    if degree not in (2, 3):
        raise ValueError("motion_blur degree must be 2 or 3")
    f32 = np.float32
    c = degree / 2
    a = angle * (3.1415926535897932384626433832795 / 180)
    al, be = math.cos(a), math.sin(a)
    m = [al, be, (1 - al) * c - be * c, -be, al, be * c + (1 - al) * c]          # getRotationMatrix2D
    d = m[0] * m[4] - m[1] * m[3]
    d = 1.0 / d if d != 0 else 0.0
    i00, i01, i10, i11 = m[4] * d, -m[1] * d, -m[3] * d, m[0] * d                # the inverse warpAffine maps with
    i02, i12 = -i00 * m[2] - i01 * m[5], -i10 * m[2] - i11 * m[5]
    k = np.zeros((degree, degree))
    for y in range(degree):
        x0, y0 = round((i01 * y + i02) * 1024) + 16, round((i11 * y + i12) * 1024) + 16    # round(): half to even, as cvRound
        for x in range(degree):
            X, Y = (x0 + round(i00 * x * 1024)) >> 5, (y0 + round(i10 * x * 1024)) >> 5
            sx, sy, vx, vy = X >> 5, Y >> 5, f32((X & 31) / 32), f32((Y & 31) / 32)
            w = ((f32(1) - vy) * (f32(1) - vx), (f32(1) - vy) * vx, vy * (f32(1) - vx), vy * vx)
            s = 0.0
            for (r, q), wk in zip(((sy, sx), (sy, sx + 1), (sy + 1, sx), (sy + 1, sx + 1)), w):
                s = s + (1.0 if r == q and 0 <= r < degree else 0.0) * float(wk)
            k[y, x] = s
    return (k / degree).astype(f32)


def augment_batch(imgs, alpha=None, beta=None, rw=None, rh=None, luts=None, out=None, blur=None):
    """img_aug (utils/datasets.py:63-68) on a CUDA uint8 [N, 3, H, W] batch, in the reference's order: contrast_and_brightness
    (alpha, beta: [N]), then motion_blur (blur: [N] of None for an image that drew no blur, or its (degree, angle)), then
    random_resize (rw, rh: [N] intermediate sizes), then augment_hsv (luts: uint8 [N, 3, 256], see hsv_luts).  A step whose
    arguments are None is skipped.  Returns a new tensor (or writes `out`; `out` may be `imgs` when there is no resize)."""
    _require_cuda(imgs, "imgs")
    if imgs.dtype != torch.uint8 or imgs.dim() != 4 or imgs.shape[1] != 3:
        raise TypeError("augment_batch expects uint8 [N, 3, H, W] images")
    imgs = imgs.contiguous()
    N, _, H, W = imgs.shape
    flags = 0
    params = (AugParams * N)()
    if alpha is not None:
        flags |= AUG_CONTRAST
        a = [float(v) for v in alpha]
        b = [float(v) for v in beta]
        if len(a) != N or len(b) != N:
            raise ValueError("one (alpha, beta) pair per image")
        for i in range(N):
            params[i].alpha, params[i].beta = a[i], b[i]
    if rw is not None:
        flags |= AUG_RESIZE
        w, h = [int(v) for v in rw], [int(v) for v in rh]
        if len(w) != N or len(h) != N:
            raise ValueError("one (rw, rh) pair per image")
        for i in range(N):
            params[i].rw, params[i].rh = w[i], h[i]
    lut_dev = None
    if luts is not None:
        flags |= AUG_HSV
        lut_dev = torch.as_tensor(luts, dtype=torch.uint8).to(imgs.device).contiguous()
        if tuple(lut_dev.shape) != (N, 3, 256):
            raise ValueError("luts must be [N, 3, 256]")
    if out is None:
        out = torch.empty_like(imgs)
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None             # noqa: E731
    with torch.cuda.device(imgs.device):
        if blur is None:
            _check(lib().yfv2_aug_batch(p(imgs), p(out), N, H, W, params, p(lut_dev), flags, _stream(imgs.device)), "aug_batch")
            return out
        if len(blur) != N:
            raise ValueError("one blur entry (None or (degree, angle)) per image")
        desc = (AugBlur * N)()
        for i, d in enumerate(blur):
            if d is not None:
                k = motion_blur_taps(int(d[0]), float(d[1]))
                desc[i].ksize = k.shape[0]
                for j, v in enumerate(k.ravel()):
                    desc[i].taps[j] = float(v)
        nb = ctypes.c_size_t()
        _check(lib().yfv2_aug_blur_workspace_bytes(N, H, W, ctypes.byref(nb)), "aug_blur_workspace_bytes")
        ws = torch.empty(nb.value, dtype=torch.uint8, device=imgs.device)
        _check(lib().yfv2_aug_batch_blur(p(imgs), p(out), N, H, W, params, p(lut_dev), desc, flags | AUG_BLUR, p(ws), nb.value,
                                         _stream(imgs.device)), "aug_batch_blur")
    return out


def _hsv_debug(fn, what, pixels, *row_w):
    """Test hook: uint8 [..., 3] CUDA pixels through the device's cv2.cvtColor conversion."""
    _require_cuda(pixels, "pixels")
    pixels = pixels.contiguous()
    out = torch.empty_like(pixels)
    with torch.cuda.device(pixels.device):
        _check(fn(ctypes.c_void_p(pixels.data_ptr()), ctypes.c_void_p(out.data_ptr()), pixels.numel() // 3, *row_w,
                  _stream(pixels.device)), what)
    return out


def debug_bgr2hsv(pixels):
    return _hsv_debug(lib().yfv2_debug_bgr2hsv, "debug_bgr2hsv", pixels)


def debug_hsv2bgr(pixels):
    """pixels [h, w, 3]: cv2.cvtColor(pixels, COLOR_HSV2BGR), which rounds the tail of each w-pixel row its own way."""
    return _hsv_debug(lib().yfv2_debug_hsv2bgr, "debug_hsv2bgr", pixels, pixels.shape[-2] if pixels.dim() >= 2 else 1)


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


def _jpeg_name(names, i):
    return str(names[i]) if names is not None else "file %d" % i


def _jpeg_pack(files, pin):
    """The files in one host uint8 tensor (pinned for an asynchronous copy when pin) and the int64 offsets of each (N + 1)."""
    import numpy as np
    arrs = []
    for i, f in enumerate(files):
        if isinstance(f, (bytes, bytearray, memoryview)):
            arrs.append(np.frombuffer(f, np.uint8))
        elif isinstance(f, np.ndarray) and f.dtype == np.uint8:
            arrs.append(np.ascontiguousarray(f).reshape(-1))
        else:
            raise Yfv2Error("decode_jpeg: file %d must be bytes or a uint8 numpy buffer, got %s" % (i, type(f).__name__))
    offsets = np.zeros(len(arrs) + 1, np.int64)
    offsets[1:] = np.cumsum([a.size for a in arrs])
    host = torch.empty(max(int(offsets[-1]), 1), dtype=torch.uint8, pin_memory=pin)
    hv = host.numpy()
    for a, o in zip(arrs, offsets):
        hv[o:o + a.size] = a
    return host, offsets


def parse_jpeg(files, names=None, blob=False, pin=False, progressive=False, strict=True):
    """yfv2_jpeg_parse_ex of files (bytes or uint8 numpy buffers), on the host only: (infos, blob, (workspace_bytes, frames_bytes),
    host buffer, offsets).  infos: one dict per file (status, w, h, components, h_samp, v_samp, orientation, restart_interval,
    segments, scans, frame_offset, reason).  Raises Yfv2Error naming every refused file and its reason; blob (a host uint8 tensor,
    pinned when pin) is None unless asked for.  progressive: accept progressive files too (flags YFV2_JPEG_PROGRESSIVE).
    strict=False: a batch with refused files returns instead of raising, with every file's status and reason in infos, blob None
    and sizes (0, 0); parse the accepted files again to decode them.  Makes no CUDA call unless pin."""
    files = list(files)
    if not files:
        raise Yfv2Error("decode_jpeg: no files")
    host, offsets = _jpeg_pack(files, pin)
    N = len(files)
    infos = (JpegInfo * N)()
    meta, ws, fr = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_size_t()
    L = lib()
    off = ctypes.c_void_p(offsets.ctypes.data)
    flags = JPEG_PROGRESSIVE if progressive else 0
    rc = L.yfv2_jpeg_parse_ex(ctypes.c_void_p(host.data_ptr()), off, N, flags, infos, None, 0, ctypes.byref(meta), ctypes.byref(ws),
                              ctypes.byref(fr))
    keys = [k for k, _ in JpegInfo._fields_]
    if rc != 0:
        bad = ["%s: %s" % (_jpeg_name(names, i), infos[i].reason.decode("utf-8", "replace")) for i in range(N) if infos[i].status]
        if not bad:
            _check(rc, "jpeg_parse")
        if not strict:
            dicts = [{k: (getattr(i, k).decode("utf-8", "replace") if k == "reason" else getattr(i, k)) for k in keys} for i in infos]
            return dicts, None, (0, 0), host, offsets
        raise Yfv2Error("decode_jpeg: %d of %d files refused: %s" % (len(bad), N, "; ".join(bad)))
    out = None
    if blob:
        out = torch.empty(meta.value, dtype=torch.uint8, pin_memory=pin)
        _check(L.yfv2_jpeg_parse_ex(ctypes.c_void_p(host.data_ptr()), off, N, flags, infos, ctypes.c_void_p(out.data_ptr()),
                                    out.numel(), ctypes.byref(meta), ctypes.byref(ws), ctypes.byref(fr)), "jpeg_parse")
    dicts = [{k: (getattr(i, k).decode() if k == "reason" else getattr(i, k)) for k in keys} for i in infos]
    return dicts, out, (ws.value, fr.value), host, offsets


class JpegBatch:
    """Files parsed on the host and copied to `device` once (one H2D copy of the packed files, one of the blob), with the workspace
    and the error flags allocated: decode() launches the three phases (or a subset) on the current stream without synchronising,
    check() waits for the flags and raises on any, frames() are [h, w, 3] uint8 views into the arena (allocated by the first
    decode()).  decode_resize(out, W, H) decodes straight into a [N, 3, H, W] network input instead, with no arena.
    progressive: accept progressive files too (parse_jpeg).  parsed: the result of parse_jpeg(files, blob=True, ...) made
    elsewhere (another process, say), used instead of parsing `files` (which may then be None)."""

    def __init__(self, files, device=None, names=None, progressive=False, parsed=None):
        device = torch.device(device if device is not None else torch.device("cuda", torch.cuda.current_device()))
        if device.type != "cuda":
            raise Yfv2Error("decode_jpeg: runs on CUDA devices only (no CPU fallback)")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        self.device, self.names = device, names
        if parsed is None:
            parsed = parse_jpeg(files, names, blob=True, pin=True, progressive=progressive)
        self.infos, self.blob, (ws_b, fr_b), host, offsets = parsed
        if self.blob is None:
            raise Yfv2Error("decode_jpeg: the parse result has no blob (parse_jpeg(..., blob=True) of accepted files)")
        self.files_bytes = int(offsets[-1])
        with torch.cuda.device(device):
            self.files = host.to(device, non_blocking=True)
            self.meta = self.blob.to(device, non_blocking=True)
            self.workspace = torch.empty(max(ws_b, 1), dtype=torch.uint8, device=device)
            self.errors = torch.zeros(len(self.infos), dtype=torch.int32, device=device)
        self.arena = None
        self._host = host                                # the pinned source of the asynchronous copy
        self._sizes = (ws_b, fr_b)

    def decode(self, phases=JPEG_ALL):
        p = lambda t: ctypes.c_void_p(t.data_ptr())     # noqa: E731
        with torch.cuda.device(self.device):
            if self.arena is None:
                self.arena = torch.empty(max(self._sizes[1], 1), dtype=torch.uint8, device=self.device)
            _check(lib().yfv2_jpeg_decode(p(self.blob), p(self.meta), self.blob.numel(), p(self.files), self.files_bytes, p(self.arena),
                                          self._sizes[1], p(self.errors), p(self.workspace), self._sizes[0], phases,
                                          _stream(self.device)), "jpeg_decode")

    def decode_resize(self, out, W, H):
        """Every file as cv2.resize(cv2.imread(f), (W, H), INTER_LINEAR) transposed to CHW, into out (a contiguous CUDA uint8
        [N, 3, H, W] tensor on the batch's device), on the current stream without synchronising; the flags as decode() sets them."""
        N = len(self.infos)
        if (not isinstance(out, torch.Tensor) or tuple(out.shape) != (N, 3, H, W) or out.dtype != torch.uint8 or not out.is_contiguous()
                or out.device != self.device):
            raise Yfv2Error("decode_resize_jpeg: out must be a contiguous uint8 tensor of shape %s on %s" % ((N, 3, H, W), self.device))
        p = lambda t: ctypes.c_void_p(t.data_ptr())     # noqa: E731
        with torch.cuda.device(self.device):
            _check(lib().yfv2_jpeg_decode_resize(p(self.blob), p(self.meta), self.blob.numel(), p(self.files), self.files_bytes, int(H),
                                                 int(W), p(out), p(self.errors), p(self.workspace), self._sizes[0],
                                                 _stream(self.device)), "jpeg_decode_resize")
        return out

    def flags(self):
        """The per-file flag words of the last decode (waits for it)."""
        return self.errors.cpu().tolist()

    def check(self):
        errs = self.flags()
        bad = [(i, e) for i, e in enumerate(errs) if e]
        if bad:
            raise Yfv2Error("decode_jpeg: %d of %d files failed to decode: %s" % (
                len(bad), len(errs), "; ".join("%s: %s" % (_jpeg_name(self.names, i), jpeg_flag_reason(e)) for i, e in bad)))

    def frames(self):
        return [self.arena[i["frame_offset"]:i["frame_offset"] + 3 * i["w"] * i["h"]].view(i["h"], i["w"], 3) for i in self.infos]


def jpeg_flag_reason(e):
    """What a yfv2_jpeg_decode flag word says, in words."""
    what = ("entropy-coded data ran out (truncated or corrupt)", "invalid Huffman code", "restart markers out of sequence")
    return ", ".join(w for b, w in enumerate(what) if e >> b & 1) or "error %d" % e


def decode_jpeg(files, device=None, names=None, progressive=False):
    """cv2.imread of JPEG files on the device: files are bytes or uint8 numpy buffers (a file's contents); returns one CUDA uint8
    [h, w, 3] BGR tensor per file, views into one arena, bit-identical to cv2.imdecode(buf, IMREAD_COLOR) / cv2.imread (EXIF
    orientation applied).  A file outside the supported subset (include/yfv2.h) raises Yfv2Error before anything is launched,
    naming it (names[i] when given) and why; so does a file whose entropy-coded data is cut short or corrupt, after the decode.
    progressive: decode progressive files too (off, they are refused as outside the subset); a progressive file cut before its
    end raises as cut short."""
    b = JpegBatch(files, device, names, progressive)
    b.decode()
    b.check()
    return b.frames()


def decode_resize_jpeg(files, W, H, device=None, names=None, progressive=False, out=None):
    """cv2.resize(cv2.imread(f), (W, H), interpolation=cv2.INTER_LINEAR) of JPEG files, transposed to the [N, 3, H, W] uint8 batch
    the network takes, in one call (yfv2_jpeg_decode_resize): bit-identical to resize_bgr(decode_jpeg(files), W, H), without the
    full-size frames.  Refuses and raises as decode_jpeg does; out: a contiguous CUDA uint8 [N, 3, H, W] tensor to write into."""
    b = JpegBatch(files, device, names, progressive)
    N = len(b.infos)
    if out is None:
        out = torch.empty((N, 3, H, W), dtype=torch.uint8, device=b.device)
    b.decode_resize(out, W, H)
    b.check()
    return out


ANCHOR_ACTIVE, ANCHOR_CONVERGED, ANCHOR_EMPTY_CLUSTER, ANCHOR_NOT_CONVERGED = 0, 1, 2, 3     # yfv2_anchor_kmeans_step status
KmeansResult = collections.namedtuple("KmeansResult", "centroids iterations status avg_iou assignments")


def kmeans_anchors(dims, k, init_idx, max_iter=1000, device=None):
    """The reference's genanchors kmeans (genanchors.py:67-102) for R runs at once on the device, bit-identical iteration by
    iteration.  dims: float64 [N, 2] box (w, h); init_idx: [R, k] box indices, run r's initial centroids dims[init_idx[r]].
    Returns CUDA tensors: centroids float64 [R, k, 2], iterations int32 [R], status int32 [R] (ANCHOR_CONVERGED, or
    ANCHOR_EMPTY_CLUSTER / ANCHOR_NOT_CONVERGED where the reference would not stop), avg_iou float64 [R] (avg_IOU of the
    centroids) and assignments int32 [R, N].  A run stopped by an empty cluster or by max_iter returns the centroids and the
    assignments of its last iteration.  One read-back of the number of active runs per iteration is the only synchronisation."""
    device = torch.device(device if device is not None else "cuda")
    X = np.ascontiguousarray(dims, dtype=np.float64)
    init = np.asarray(init_idx, dtype=np.int64)
    if X.ndim != 2 or X.shape[1] != 2 or init.ndim != 2 or init.shape[1] != k:
        raise Yfv2Error("kmeans_anchors: dims must be [N, 2] and init_idx [R, k=%d], got %s and %s" % (k, X.shape, init.shape))
    N, R = X.shape[0], init.shape[0]
    if N and init.size and (init.min() < 0 or init.max() >= N):
        raise Yfv2Error("kmeans_anchors: init_idx holds indices outside [0, %d)" % N)
    boxes = torch.from_numpy(X).to(device)
    cent = torch.from_numpy(np.ascontiguousarray(X[init] if N and init.size else np.zeros((R, k, 2)))).to(device)
    assignments = torch.full((R, N), -1, dtype=torch.int32, device=device)
    iterations = torch.zeros(R, dtype=torch.int32, device=device)
    status = torch.zeros(R, dtype=torch.int32, device=device)
    changed = torch.zeros(R, dtype=torch.int32, device=device)
    active = torch.zeros(1, dtype=torch.int32, device=device)
    active_host = torch.zeros(1, dtype=torch.int32).pin_memory()
    avg = torch.empty(R, dtype=torch.float64, device=device)
    L, s = lib(), _stream(device)
    with torch.cuda.device(device):
        while True:
            _check(L.yfv2_anchor_kmeans_step(boxes.data_ptr(), N, k, R, max_iter, cent.data_ptr(), assignments.data_ptr(),
                                             iterations.data_ptr(), status.data_ptr(), changed.data_ptr(), active.data_ptr(), s),
                   "anchor_kmeans_step")
            active_host.copy_(active, non_blocking=True)
            torch.cuda.current_stream(device).synchronize()
            if active_host.item() == 0:
                break
        _check(L.yfv2_anchor_avg_iou(boxes.data_ptr(), N, k, R, cent.data_ptr(), avg.data_ptr(), s), "anchor_avg_iou")
    return KmeansResult(cent, iterations, status, avg, assignments)


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


# cv2's IMWRITE_* ids and IMWRITE_JPEG_SAMPLING_FACTOR_* values (yfv2_jpeg_encode_plan reads the same pairs)
IMWRITE_JPEG_QUALITY, IMWRITE_JPEG_PROGRESSIVE, IMWRITE_JPEG_OPTIMIZE, IMWRITE_JPEG_RST_INTERVAL = 1, 2, 3, 4
IMWRITE_JPEG_LUMA_QUALITY, IMWRITE_JPEG_CHROMA_QUALITY, IMWRITE_JPEG_SAMPLING_FACTOR = 5, 6, 7
JPEG_SAMPLING = {"420": 0x221111, "422": 0x211111, "444": 0x111111, "440": 0x121111, "411": 0x411111}
_ENC_KIND = {"bgr": 0, "strided": 1, "gray": 2, "yuv420": 3, "yuv422": 4}


def _enc_frame(f, lay, device, d, keep):
    """Fills d (a JpegEncSrc) with the descriptor of checked frame f in layout `lay`, its pixels on `device`; returns (h, w)."""
    kind = "gray" if lay == "gray" else _KIND[lay]
    d.kind = _ENC_KIND[kind]
    if kind == "bgr":
        f = _frame_on_device(f, device)
        d.f.bgr.data, d.f.bgr.w, d.f.bgr.h, d.f.bgr.pitch = f.data_ptr(), f.shape[1], f.shape[0], f.stride(0)
        keep.append(f)
        return f.shape[0], f.shape[1]
    if kind == "yuv420":
        y, u, v = [p.to(device) for p in _yuv420_planes(f, lay, 0)]
        y, u, v = [p if p.stride(1) == 1 else p.contiguous() for p in (y, u, v)]
        e = d.f.yuv420
        if lay in ("nv12", "nv21"):
            e.u, e.v, e.uv_pitch, e.uv_step = u.data_ptr() + (lay == "nv21"), u.data_ptr() + (lay == "nv12"), u.stride(0), 2
        else:
            if u.stride(0) != v.stride(0):
                u, v = u.contiguous(), v.contiguous()
            e.u, e.v, e.uv_pitch, e.uv_step = u.data_ptr(), v.data_ptr(), u.stride(0), 1
        e.y, e.y_pitch, e.h, e.w = y.data_ptr(), y.stride(0), y.shape[0], y.shape[1]
        keep += [y, u, v]
        return e.h, e.w
    f = f.to(device)
    if lay == "rgb_chw":
        if f.stride(2) != 1 or f.stride(1) < f.shape[2]:
            f = f.contiguous()
        p, s = f.data_ptr(), f.stride(0)
        e = d.f.strided
        e.b, e.g, e.r, e.pitch, e.step, e.h, e.w = p + 2 * s, p + s, p, f.stride(1), 1, f.shape[1], f.shape[2]
        keep.append(f)
        return e.h, e.w
    step = 1 if lay == "gray" else _CHANNELS[lay]
    if f.stride(1) != step or (lay != "gray" and f.stride(2) != 1) or f.stride(0) < step * f.shape[1]:
        f = f.contiguous()
    p = f.data_ptr()
    if kind == "yuv422":
        e = d.f.yuv422
        oy, ou, ov = _YUV422_OFFSETS[lay]
        e.y, e.u, e.v = p + oy, p + ou, p + ov
    else:
        e = d.f.strided
        ob, og, or_ = _BGR_OFFSETS[lay]
        e.b, e.g, e.r, e.step = p + ob, p + og, p + or_, step
    e.pitch, e.h, e.w = f.stride(0), f.shape[0], f.shape[1]
    keep.append(f)
    return e.h, e.w


def _per_output(v, n, what):
    v = list(v) if isinstance(v, (list, tuple)) else [v] * n
    if len(v) != n:
        raise Yfv2Error("encode_jpeg: %d values of %s for %d outputs" % (len(v), what, n))
    return v


def encode_jpeg(frames, quality=95, sampling="420", restart_interval=0, layout="bgr", regions=None, device=None, params=None,
                device_out=False):
    """cv2.imencode('.jpg', img, params)[1] of every output, byte for byte (OpenCV 4.13), encoded on the device in one call
    (yfv2_jpeg_encode).  img is cv2.cvtColor(frame, COLOR_<LAYOUT>2BGR) for any layout of resize_frames (one name, or one per
    frame); "gray" frames give one-component JPEGs, as cv2 does for a 2-D array.  regions: None (one output per frame, the whole
    frame), or a list of (frame index, x0, y0, w, h), one output each, cropped from the converted frame (several may share a
    frame).  quality (any int, clamped to 0..100 as cv2 does), sampling ("420", "422", "444") and restart_interval (MCUs, 0: none)
    are one value or one per output; params: extra cv2 (IMWRITE_*, value) pairs for every output, or a list of them per output.
    Everything is checked before anything is launched; a refusal raises Yfv2Error naming the output.  Returns a list of bytes, or
    with device_out=True (arena, offsets, lengths): the uint8 CUDA arena, output i at offsets[i] (host int64 numpy) and
    lengths[i] bytes long (CUDA int64), with no copy to the host."""
    import numpy as np
    frames = list(frames)
    layouts = [layout] * len(frames) if isinstance(layout, str) else list(layout)
    if not frames:
        raise Yfv2Error("encode_jpeg: no frames")
    if len(layouts) != len(frames):
        raise Yfv2Error("encode_jpeg: %d layouts for %d frames" % (len(layouts), len(frames)))
    for lay in layouts:
        if not isinstance(lay, str) or lay not in LAYOUTS:
            raise Yfv2Error("encode_jpeg: layout must be one of %s, got %r" % (", ".join(LAYOUTS), lay))
    checked = [_check_frame(f, lay, i) for i, (f, lay) in enumerate(zip(frames, layouts))]
    if regions is None:
        regions = [(i, 0, 0, None, None) for i in range(len(frames))]
    regions = [tuple(r) for r in regions]
    n = len(regions)
    if n == 0:
        raise Yfv2Error("encode_jpeg: no regions")
    for k, r in enumerate(regions):
        if len(r) != 5 or not 0 <= int(r[0]) < len(frames):
            raise Yfv2Error("encode_jpeg: region %d must be (frame index in [0, %d), x0, y0, w, h), got %r" % (k, len(frames), r))
    qs, ss, rs = _per_output(quality, n, "quality"), _per_output(sampling, n, "sampling"), _per_output(restart_interval, n, "restart")
    extra = params if params and isinstance(params[0], (list, tuple)) else [params or []] * n
    if len(extra) != n:
        raise Yfv2Error("encode_jpeg: %d params lists for %d outputs" % (len(extra), n))
    plist = []
    for k in range(n):
        if ss[k] not in JPEG_SAMPLING:
            raise Yfv2Error("encode_jpeg: output %d: sampling must be one of %s, got %r" % (k, ", ".join(JPEG_SAMPLING), ss[k]))
        plist.append([IMWRITE_JPEG_QUALITY, int(qs[k]), IMWRITE_JPEG_SAMPLING_FACTOR, JPEG_SAMPLING[ss[k]],
                      IMWRITE_JPEG_RST_INTERVAL, int(rs[k])] + [int(x) for x in extra[k]])
    if device is None:
        cuda = [t.device for f in checked for t in (f if isinstance(f, (tuple, list)) else (f,))
                if isinstance(t, torch.Tensor) and t.is_cuda]
        device = cuda[0] if cuda else torch.device("cuda", torch.cuda.current_device())
    device = torch.device(device)
    if device.type != "cuda":
        raise Yfv2Error("encode_jpeg: runs on CUDA devices only (no CPU fallback)")
    srcs = (JpegEncSrc * n)()
    keep, cparams, frame_desc = [], [], {}
    for k, (d, r) in enumerate(zip(srcs, regions)):
        i = int(r[0])
        if i not in frame_desc:
            frame_desc[i] = JpegEncSrc()
            frame_desc[i].hw = _enc_frame(checked[i], layouts[i], device, frame_desc[i], keep)
        src = frame_desc[i]
        d.kind, d.f = src.kind, src.f
        fh, fw = src.hw
        d.x0, d.y0 = int(r[1]), int(r[2])
        d.w = fw if r[3] is None else int(r[3])
        d.h = fh if r[4] is None else int(r[4])
        pa = (ctypes.c_int * len(plist[k]))(*plist[k])
        cparams.append(pa)
        d.params, d.nparams = ctypes.cast(pa, ctypes.POINTER(ctypes.c_int)), len(plist[k])
    L = lib()
    meta_b, ws_b, arena_b = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_size_t()
    offsets = np.zeros(n + 1, np.int64)
    off_p = offsets.ctypes.data_as(ctypes.POINTER(ctypes.c_longlong))
    _check(L.yfv2_jpeg_encode_plan(srcs, n, None, 0, ctypes.byref(meta_b), ctypes.byref(ws_b), off_p, ctypes.byref(arena_b)),
           "jpeg_encode_plan")
    meta = torch.empty(meta_b.value, dtype=torch.uint8, pin_memory=True)
    _check(L.yfv2_jpeg_encode_plan(srcs, n, ctypes.c_void_p(meta.data_ptr()), meta_b.value, ctypes.byref(meta_b),
                                   ctypes.byref(ws_b), off_p, ctypes.byref(arena_b)), "jpeg_encode_plan")
    with torch.cuda.device(device):
        meta_dev = meta.to(device, non_blocking=True)
        ws = torch.empty(ws_b.value, dtype=torch.uint8, device=device)
        arena = torch.empty(arena_b.value, dtype=torch.uint8, device=device)
        lengths = torch.empty(n, dtype=torch.int64, device=device)
        _check(L.yfv2_jpeg_encode(ctypes.c_void_p(meta.data_ptr()), ctypes.c_void_p(meta_dev.data_ptr()), meta_b.value,
                                  ctypes.c_void_p(ws.data_ptr()), ws_b.value, ctypes.c_void_p(arena.data_ptr()), arena_b.value,
                                  ctypes.c_void_p(lengths.data_ptr()), 15, _stream(device)), "jpeg_encode")
        if device_out:
            torch.cuda.current_stream(device).synchronize()   # the host blob and the frames' copies stay alive until it ran
            return arena, offsets[:n], lengths
        lens = lengths.cpu().numpy()
        # only the bytes written come back: each output's slot is its worst case, usually far larger than the file
        return [arena[int(offsets[k]):int(offsets[k]) + int(lens[k])].cpu().numpy().tobytes() for k in range(n)]


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
    N, h, w, A, C = head_geometry("export_heads", preds)
    preds = [p.detach().contiguous().float() for p in preds]
    dev = preds[0].device
    o2 = torch.empty((N, h, w, 5 * A + C), dtype=torch.float32, device=dev)
    o3 = torch.empty((N, h // 2, w // 2, 5 * A + C), dtype=torch.float32, device=dev)
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
    _require_cuda(out2, "ncnn_post: out2")
    if out2.dim() != 4 or out2.shape[1] % 2 or out2.shape[2] % 2 or out2.shape[1] == 0 or out2.shape[2] == 0:
        raise Yfv2Error("ncnn_post: out2 has shape %s, expected [N, H/16, W/16, 5A+C] with H, W multiples of 32" % (tuple(out2.shape),))
    N, h, w, ch = out2.shape
    _expect_shapes("ncnn_post", [out2, out3], ["out2", "out3"], [(N, h, w, ch), (N, h // 2, w // 2, ch)])
    out2 = out2.detach().contiguous().float(); out3 = out3.detach().contiguous().float()
    A = int(anchor_num)
    C = ch - 5 * A
    H, W = h * 16, w * 16
    M = A * (h * w + (h // 2) * (w // 2))
    max_out = M if max_out is None else int(max_out)
    if max_out < 1:
        raise Yfv2Error("ncnn_post: max_out=%d, expected at least 1" % max_out)
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

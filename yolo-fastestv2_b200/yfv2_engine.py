"""ctypes binding of libyfv2.so (include/yfv2.h) plus the small amount of host bookkeeping the Python
mirror modules share: plan cache, weight packing, output allocation.  PyTorch is used for device
memory and streams only; every device computation is a kernel inside libyfv2.so.

There is NO CPU fallback: if the library is missing or the tensors are not on a CUDA device the calls
raise.
"""
import collections
import contextlib
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


class BayerFrame(ctypes.Structure):
    """yfv2_bayer_frame: the window (x0, y0, w, h) of the demosaic of a whole raw Bayer frame in device memory."""
    _fields_ = [("data", ctypes.c_void_p), ("pitch", ctypes.c_longlong), ("fw", ctypes.c_int), ("fh", ctypes.c_int),
                ("x0", ctypes.c_int), ("y0", ctypes.c_int), ("w", ctypes.c_int), ("h", ctypes.c_int), ("red_x", ctypes.c_int),
                ("red_y", ctypes.c_int), ("edge_aware", ctypes.c_int)]


class _EncFrame(ctypes.Union):
    _fields_ = [("bgr", Frame), ("strided", StridedFrame), ("yuv420", Yuv420Frame), ("yuv422", Yuv422Frame),
                ("bayer", BayerFrame)]


class JpegEncSrc(ctypes.Structure):
    """yfv2_jpeg_enc_src: one output of yfv2_jpeg_encode: a frame, its region and cv2.imencode's params."""
    _fields_ = [("kind", ctypes.c_int), ("x0", ctypes.c_int), ("y0", ctypes.c_int), ("w", ctypes.c_int), ("h", ctypes.c_int),
                ("f", _EncFrame), ("params", ctypes.POINTER(ctypes.c_int)), ("nparams", ctypes.c_int)]


# JpegEncSrc.kind (YFV2_JPEG_SRC_*)
JPEG_SRC_BGR, JPEG_SRC_STRIDED, JPEG_SRC_GRAY, JPEG_SRC_YUV420, JPEG_SRC_YUV422, JPEG_SRC_BAYER = range(6)


class RemapMap(ctypes.Structure):
    """yfv2_remap_map: cv2's fixed remap maps in device memory, xy (CV_16SC2) and code (CV_16UC1)."""
    _fields_ = [("xy", ctypes.c_void_p), ("xy_pitch", ctypes.c_longlong), ("code", ctypes.c_void_p),
                ("code_pitch", ctypes.c_longlong), ("mw", ctypes.c_int), ("mh", ctypes.c_int)]


class RemapFrame(ctypes.Structure):
    """yfv2_remap_frame: the window (x0, y0, w, h) of cv2.remap of an inner frame (kind: YFV2_JPEG_SRC_*, not GRAY)."""
    _fields_ = [("kind", ctypes.c_int), ("x0", ctypes.c_int), ("y0", ctypes.c_int), ("w", ctypes.c_int), ("h", ctypes.c_int),
                ("f", _EncFrame), ("map", RemapMap)]


class WarpFrame(ctypes.Structure):
    """yfv2_warp_frame: the window (x0, y0, w, h) of cv2.warpAffine / cv2.warpPerspective (dsize dw x dh) of an inner frame."""
    _fields_ = [("kind", ctypes.c_int), ("x0", ctypes.c_int), ("y0", ctypes.c_int), ("w", ctypes.c_int), ("h", ctypes.c_int),
                ("f", _EncFrame), ("m", ctypes.c_double * 9), ("perspective", ctypes.c_int), ("inverse", ctypes.c_int),
                ("dw", ctypes.c_int), ("dh", ctypes.c_int)]


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


class TrainLaunchRecord(ctypes.Structure):
    """yfv2_train_launch: one kernel launch or memset of a training operator or a native training step (test hook)."""
    _fields_ = [("kernel", ctypes.c_char * 32), ("op", ctypes.c_int), ("bwd", ctypes.c_int), ("grid", ctypes.c_int * 3), ("block", ctypes.c_int),
                ("smem", ctypes.c_longlong), ("bytes", ctypes.c_longlong)] + \
               [(f, ctypes.c_int) for f in ("bm", "vec_b", "vec_c", "vec", "pchunk", "chunks", "partial", "slices", "accumulate")]


TRAIN_OPS = ("conv1x1_fwd", "conv1x1_bwd", "dwconv_fwd", "dwconv_bwd", "stem_fwd", "stem_wgrad", "bn_train_fwd", "bn_train_bwd",
             "bn_eval_fwd", "bn_eval_bwd", "maxpool_fwd", "maxpool_bwd", "upsample2_fwd", "upsample2_bwd")     # YFV2_OP_*


def _train_launches(call, what):
    n = ctypes.c_int()
    _check(call(None, 0, ctypes.byref(n)), what)
    recs = (TrainLaunchRecord * n.value)()
    _check(call(recs, n.value, ctypes.byref(n)), what)
    names = [f for f, _ in TrainLaunchRecord._fields_]
    out = []
    for r in recs:
        d = {f: getattr(r, f) for f in names}
        d["kernel"], d["grid"], d["bwd"] = r.kernel.decode(), tuple(r.grid), bool(r.bwd)
        out.append(d)
    return out


def trainer_launches(handle, workspace=None, sms=0):
    """The kernel launches and memsets of one training step of a yfv2_trainer handle under its current mode (forward, then backward
    with accumulate = 0), in order, as dicts (yfv2_trainer_debug_launches; host only).  workspace None: a 16-byte-aligned workspace;
    sms 0: this device's SM count."""
    L, ws = lib(), ctypes.c_void_p(workspace)
    return _train_launches(lambda out, cap, n: L.yfv2_trainer_debug_launches(handle, ws, sms, out, cap, n), "trainer_debug_launches")


def op_launches(name, ptrs, ints, sms=0):
    """The kernel launches and memsets of one yfv2_op_<name> call, in order, as dicts (yfv2_op_debug_launches; host only).  ptrs: the
    call's pointer arguments as integer addresses (None: NULL), ints: its integer arguments, both in signature order."""
    args = PROTOTYPES["yfv2_op_" + name][1][:-1]                         # the call's arguments without the stream
    want = (sum(a is ctypes.c_void_p for a in args), sum(a is ctypes.c_int for a in args))
    if (len(ptrs), len(ints)) != want:
        raise Yfv2Error("op_launches: yfv2_op_%s takes %d pointers and %d integers, got %d and %d" % ((name,) + want + (len(ptrs), len(ints))))
    L = lib()
    p = (ctypes.c_void_p * len(ptrs))(*ptrs)
    i = (ctypes.c_int * len(ints))(*ints)
    return _train_launches(lambda out, cap, n: L.yfv2_op_debug_launches(TRAIN_OPS.index(name), p, i, sms, out, cap, n), "op_debug_launches")


_dispatch = [(0, 0)]         # the (sms, ctas) simulated_dispatch last set (the library's setting is process-wide)


@contextlib.contextmanager
def simulated_dispatch(sms=0, ctas=0):
    """Within the block, launches are chosen as on a GPU of `sms` SMs, and a persistent forward launch runs exactly min(items, ctas)
    CTAs (yfv2_debug_set_dispatch; 0 leaves a setting off).  The setting holds for every thread of the process, the autograd
    engine's included.  The previous setting is restored on exit, also when the block raises."""
    L, prev = lib(), _dispatch[0]
    _check(L.yfv2_debug_set_dispatch(sms, ctas), "debug_set_dispatch")
    _dispatch[0] = (sms, ctas)
    try:
        yield
    finally:
        _check(L.yfv2_debug_set_dispatch(*prev), "debug_set_dispatch")
        _dispatch[0] = prev


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
COUNT_MAX_LINES, COUNT_MAX_ZONES, COUNT_MAX_VERTICES = 32, 16, 64
COUNT_LINE, COUNT_ENTRY, COUNT_EXIT = 0, 1, 2           # kind of a yfv2_count_update event


class AugParams(ctypes.Structure):
    """yfv2_aug_params: one image's contrast (alpha, beta) and random_resize size (rw, rh)."""
    _fields_ = [("alpha", ctypes.c_float), ("beta", ctypes.c_float), ("rw", ctypes.c_int), ("rh", ctypes.c_int)]


AUG_CONTRAST, AUG_RESIZE, AUG_HSV = 1, 2, 4          # yfv2_aug_batch flags (include/yfv2.h)
AUG_BLUR = 8                                         # yfv2_aug_batch_blur adds motion_blur


class AugBlur(ctypes.Structure):
    """yfv2_aug_blur: one image's motion_blur kernel (ksize 0: the image drew no blur)."""
    _fields_ = [("ksize", ctypes.c_int), ("taps", ctypes.c_float * 9)]


class AugGeom(ctypes.Structure):
    """yfv2_aug_geom: one image's mosaic canvas, random_perspective matrix (canvas -> output) and fliplr."""
    _fields_ = [("m", ctypes.c_double * 9), ("perspective", ctypes.c_int), ("mosaic", ctypes.c_int), ("src", ctypes.c_int * 4),
                ("xc", ctypes.c_int), ("yc", ctypes.c_int), ("flip", ctypes.c_int)]


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
    "yfv2_merge_regions_nmm": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(Region), ctypes.c_int, ctypes.c_int,
                                              ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.c_int, ctypes.c_int,
                                              ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "yfv2_track_state_bytes": (ctypes.c_int, [ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_size_t)]),
    "yfv2_track_reset": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_int), ctypes.c_int,
                                        ctypes.c_void_p]),
    "yfv2_track_update": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_int), ctypes.c_int,
                                         ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(TrackParams), ctypes.c_void_p,
                                         ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "yfv2_track_debug_read": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_int),
                                             ctypes.POINTER(ctypes.c_int), ctypes.POINTER(TrackRecord), ctypes.POINTER(ctypes.c_int),
                                             ctypes.c_void_p]),
    "yfv2_count_state_bytes": (ctypes.c_int, [ctypes.c_int] * 5 + [ctypes.POINTER(ctypes.c_size_t)]),
    "yfv2_count_reset": (ctypes.c_int, [ctypes.c_void_p] + [ctypes.c_int] * 5 + [ctypes.POINTER(ctypes.c_int), ctypes.c_int,
                                                                                 ctypes.c_void_p]),
    "yfv2_count_set_geometry": (ctypes.c_int, [ctypes.c_void_p] + [ctypes.c_int] * 6 + [ctypes.POINTER(ctypes.c_double), ctypes.c_int,
                                                                                        ctypes.POINTER(ctypes.c_float),
                                                                                        ctypes.POINTER(ctypes.c_int), ctypes.c_int,
                                                                                        ctypes.c_void_p]),
    "yfv2_count_update": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p] + [ctypes.c_int] * 5 + [ctypes.POINTER(ctypes.c_int),
                                                                                                   ctypes.c_int, ctypes.c_int,
                                                                                                   ctypes.c_void_p, ctypes.c_void_p,
                                                                                                   ctypes.c_void_p, ctypes.c_void_p]),
    "yfv2_count_debug_read": (ctypes.c_int, [ctypes.c_void_p] + [ctypes.c_int] * 6 + [ctypes.POINTER(ctypes.c_int),
                                                                                      ctypes.POINTER(ctypes.c_longlong),
                                                                                      ctypes.POINTER(ctypes.c_int),
                                                                                      ctypes.POINTER(ctypes.c_double),
                                                                                      ctypes.POINTER(ctypes.c_byte),
                                                                                      ctypes.POINTER(ctypes.c_uint), ctypes.c_void_p]),
    "yfv2_batch_statistics": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                             ctypes.c_int, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p]),
    "yfv2_aug_contrast_brightness": (ctypes.c_int, [ctypes.c_void_p] * 4 + [ctypes.c_int, ctypes.c_longlong, ctypes.c_void_p]),
    "yfv2_aug_batch": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                      ctypes.POINTER(AugParams), ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]),
    "yfv2_aug_blur_workspace_bytes": (ctypes.c_int, [ctypes.c_int] * 3 + [ctypes.POINTER(ctypes.c_size_t)]),
    "yfv2_aug_batch_blur": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                           ctypes.POINTER(AugParams), ctypes.c_void_p, ctypes.POINTER(AugBlur), ctypes.c_int,
                                           ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "yfv2_aug_geometric": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                          ctypes.POINTER(AugGeom), ctypes.c_void_p]),
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
    "yfv2_resize_bayer_u8": (ctypes.c_int, [ctypes.POINTER(BayerFrame), ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                            ctypes.c_void_p]),
    "yfv2_resize_remap_u8": (ctypes.c_int, [ctypes.POINTER(RemapFrame), ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                            ctypes.c_void_p]),
    "yfv2_remap_u8": (ctypes.c_int, [ctypes.POINTER(RemapFrame), ctypes.c_int, ctypes.POINTER(ctypes.c_void_p), ctypes.c_void_p]),
    "yfv2_resize_warp_u8": (ctypes.c_int, [ctypes.POINTER(WarpFrame), ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                           ctypes.c_void_p]),
    "yfv2_warp_u8": (ctypes.c_int, [ctypes.POINTER(WarpFrame), ctypes.c_int, ctypes.POINTER(ctypes.c_void_p), ctypes.c_void_p]),
    "yfv2_warp_matrix": (ctypes.c_int, [ctypes.POINTER(WarpFrame), ctypes.POINTER(ctypes.c_double)]),
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
    "yfv2_debug_set_dispatch": (ctypes.c_int, [ctypes.c_int, ctypes.c_int]),
    "yfv2_op_debug_launches": (ctypes.c_int, [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                              ctypes.POINTER(ctypes.c_int)]),
    "yfv2_trainer_debug_launches": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                                   ctypes.POINTER(ctypes.c_int)]),
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
MERGE_MODES = ("nms", "nmm")


def merge_regions(dets, counts, regions, F, W, H, thr, metric, max_det, mode="nms", want_merged=False):
    """yfv2_merge_regions: the NMS rows of T region images -> one list per frame in frame pixels (a cross-region NMS, see
    include/yfv2.h).  dets: CUDA float32 [T, max_det_in, 6] and counts int32 [T], as decode_nms / nms return them for the region
    images; regions: T tuples (frame, x0, y0, w, h), the regions of one frame contiguous, frames ascending; F frames; W x H the
    network input the regions were stretched to; metric "iou" | "ios" (or 0 | 1).  Returns CUDA tensors (out float64
    [F, max_det, 6], counts int32 [F], kept_src int32 [F, max_det]: t * max_det_in + row of each kept row, -1 past the count).
    mode "nmm" runs yfv2_merge_regions_nmm instead: the same rows, counts and kept_src, with each kept box grown to the union of
    the rows it absorbed (greedy non-maximum merging).  want_merged (nmm only) appends a fourth tensor, int32 [F, max_det]: how
    many rows each kept box absorbed (0 past the count)."""
    if mode not in MERGE_MODES:
        raise Yfv2Error("merge_regions: mode must be 'nms' or 'nmm', got %r" % (mode,))
    if want_merged and mode != "nmm":
        raise Yfv2Error("merge_regions: want_merged needs mode='nmm'")
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
    merged = torch.empty((max(F, 0), max_det), dtype=torch.int32, device=dev) if want_merged else None
    with torch.cuda.device(dev):
        args = (ctypes.c_void_p(dets.data_ptr()), ctypes.c_void_p(counts.data_ptr()), descs, T, max_det_in, F, H, W,
                ctypes.c_double(thr), m, max_det, ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(out_counts.data_ptr()),
                ctypes.c_void_p(kept.data_ptr()))
        if mode == "nmm":
            _check(lib().yfv2_merge_regions_nmm(*args, ctypes.c_void_p(merged.data_ptr()) if want_merged else None, _stream(dev)),
                   "merge_regions_nmm")
        else:
            _check(lib().yfv2_merge_regions(*args, _stream(dev)), "merge_regions")
    return (out, out_counts, kept, merged) if want_merged else (out, out_counts, kept)


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
        """Clears the given streams (all by default, in calls of at most TRACK_MAX_BATCH streams): no tracks, frame 0, next id 1."""
        calls = [range(b, min(b + TRACK_MAX_BATCH, self.S)) for b in range(0, self.S, TRACK_MAX_BATCH)] if streams is None else [streams]
        for part in calls:
            idx, arr = self._streams(part, self.S)
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


class Counter:
    """Line crossings and zone occupancy of a Tracker's tracks (yfv2_count_*, include/yfv2.h), for every stream of the tracker.
    A track's anchor is the bottom centre of its box; a line is a directed segment (ax, ay, bx, by) and a crossing's dir is the
    side of the line the anchor ends on (+1: left of A -> B in image coordinates, y down); a zone is a polygon of 3..max_vertices
    vertices, rounded to float32, tested as cv2.pointPolygonTest tests it (the boundary is inside).  It owns the device state
    tensor; `lines` / `zones` given here apply to every stream, set_geometry gives one stream its own.  After Tracker.reset of
    some streams (their ids start again at 1), reset the same streams here."""

    def __init__(self, tracker, lines=None, zones=None, max_lines=8, max_zones=8, max_vertices=32):
        self.tracker = tracker
        self.device = tracker.device
        self.S, self.K = tracker.S, tracker.K
        self.L, self.Z, self.P = int(max_lines), int(max_zones), int(max_vertices)
        nb = ctypes.c_size_t()
        _check(lib().yfv2_count_state_bytes(self.S, self.K, self.L, self.Z, self.P, ctypes.byref(nb)), "Counter")
        geom = self._geometry(lines, zones, "Counter") if lines is not None or zones is not None else None
        self.state = torch.zeros((nb.value,), dtype=torch.uint8, device=self.device)
        if geom is not None:
            for s in range(self.S):
                self._set(s, geom, "Counter")

    def _geometry(self, lines, zones, what):
        ln = np.ascontiguousarray(np.asarray([] if lines is None else lines, np.float64).reshape(-1, 4))
        if len(ln) > self.L:
            raise Yfv2Error("%s: %d lines, max_lines=%d" % (what, len(ln), self.L))
        zs = [np.asarray(z) for z in ([] if zones is None else zones)]
        if len(zs) > self.Z:
            raise Yfv2Error("%s: %d zones, max_zones=%d" % (what, len(zs), self.Z))
        zf = np.zeros((max(len(zs), 1), self.P, 2), np.float32)
        nv = np.zeros((max(len(zs), 1),), np.int32)
        for z, v in enumerate(zs):
            if v.ndim != 2 or v.shape[1] != 2 or not 3 <= v.shape[0] <= self.P:
                raise Yfv2Error("%s: zones[%d] must be [n, 2] with n in 3..max_vertices=%d, got %s" % (what, z, self.P, tuple(v.shape)))
            zf[z, :len(v)] = v.astype(np.float32)
            nv[z] = len(v)
        return ln, zf, nv, len(zs)

    def _set(self, s, geom, what):
        ln, zf, nv, nz = geom
        with torch.cuda.device(self.device):
            _check(lib().yfv2_count_set_geometry(ctypes.c_void_p(self.state.data_ptr()), self.S, self.K, self.L, self.Z, self.P, int(s),
                                                 ln.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), len(ln),
                                                 zf.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
                                                 nv.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), nz, _stream(self.device)), what)

    def set_geometry(self, stream, lines=None, zones=None):
        """Stream `stream`'s lines [n, 4] and zones (a list of [n, 2] polygons); clears its records and totals."""
        if not 0 <= int(stream) < self.S:
            raise Yfv2Error("Counter.set_geometry: stream %d outside [0, %d)" % (int(stream), self.S))
        self._set(int(stream), self._geometry(lines, zones, "Counter.set_geometry"), "Counter.set_geometry")

    def _streams(self, streams):
        idx = list(range(self.S)) if streams is None else [int(s) for s in streams]
        return idx, (ctypes.c_int * max(len(idx), 1))(*idx)

    def reset(self, streams=None):
        """Clears the records and totals of the given streams (all by default), keeping their geometry."""
        calls = [range(b, min(b + TRACK_MAX_BATCH, self.S)) for b in range(0, self.S, TRACK_MAX_BATCH)] if streams is None else [streams]
        for part in calls:
            idx, arr = self._streams(part)
            with torch.cuda.device(self.device):
                _check(lib().yfv2_count_reset(ctypes.c_void_p(self.state.data_ptr()), self.S, self.K, self.L, self.Z, self.P, arr, len(idx),
                                              _stream(self.device)), "Counter.reset")

    def update(self, streams=None, max_events=64):
        """Counts the tracker's current frame of the given streams (None: all, at most TRACK_MAX_BATCH) in one launch without a
        host synchronisation.  Returns CUDA tensors (events float64 [B, max_events, 8]: (kind, index, dir, track_id, cls, x, y,
        frame) in ascending track id, then line, then zone order, zeros past the count; event_counts int32 [B]: every event,
        possibly more than max_events; occupancy int32 [B, max_zones])."""
        if (self.tracker.S, self.tracker.K) != (self.S, self.K):
            raise Yfv2Error("Counter.update: the tracker has S=%d K=%d, the counter S=%d K=%d" % (self.tracker.S, self.tracker.K, self.S, self.K))
        E = int(max_events)
        if E < 0:
            raise Yfv2Error("Counter.update: max_events=%d must be >= 0" % E)
        idx, arr = self._streams(streams)
        B = len(idx)
        events = torch.empty((B, E, 8), dtype=torch.float64, device=self.device)
        counts = torch.empty((B,), dtype=torch.int32, device=self.device)
        occupancy = torch.empty((B, self.Z), dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            _check(lib().yfv2_count_update(ctypes.c_void_p(self.tracker.state.data_ptr()), ctypes.c_void_p(self.state.data_ptr()), self.S,
                                           self.K, self.L, self.Z, self.P, arr, B, E, ctypes.c_void_p(events.data_ptr() if E else None),
                                           ctypes.c_void_p(counts.data_ptr()), ctypes.c_void_p(occupancy.data_ptr() if self.Z else None),
                                           _stream(self.device)), "Counter.update")
        return events, counts, occupancy

    def _read(self, stream):
        geom = (ctypes.c_int * 2)()
        totals = np.zeros((2 * self.L + 2 * self.Z,), np.int64)
        ids = np.zeros((self.K,), np.int32)
        anchors = np.zeros((self.K, 2), np.float64)
        sides = np.zeros((self.K, max(self.L, 1)), np.int8)
        inside = np.zeros((self.K,), np.uint32)
        with torch.cuda.device(self.device):
            _check(lib().yfv2_count_debug_read(ctypes.c_void_p(self.state.data_ptr()), self.S, self.K, self.L, self.Z, self.P, int(stream),
                                               geom, totals.ctypes.data_as(ctypes.POINTER(ctypes.c_longlong)),
                                               ids.ctypes.data_as(ctypes.POINTER(ctypes.c_int)),
                                               anchors.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                                               sides.ctypes.data_as(ctypes.POINTER(ctypes.c_byte)),
                                               inside.ctypes.data_as(ctypes.POINTER(ctypes.c_uint)), _stream(self.device)), "Counter")
        return geom[0], geom[1], totals, ids, anchors, sides, inside

    def totals(self, stream):
        """Stream `stream`'s running totals on the host (synchronises): {"lines": int64 [n_lines, 2] (crossings with dir +1, -1),
        "zones": int64 [n_zones, 2] (entries, exits)}."""
        nl, nz, totals = self._read(stream)[:3]
        return {"lines": totals[:2 * nl].reshape(nl, 2), "zones": totals[2 * self.L:2 * self.L + 2 * nz].reshape(nz, 2)}

    def records(self, stream):
        """Test hook (synchronises): the record of every slot that holds one, {track id: (anchor (x, y), sides [n_lines], inside
        bits)}; a slot's record outlives its track until the slot's next track appears."""
        nl, nz, _, ids, anchors, sides, inside = self._read(stream)
        return {int(i): ((float(anchors[k, 0]), float(anchors[k, 1])), sides[k, :nl].tolist(), int(inside[k]))
                for k, i in enumerate(ids) if i != 0}


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


def geom_descriptors(params):
    """The yfv2_aug_geom array of augment_geometric's params (dicts with M, perspective, mosaic, src, xc, yc, flip)."""
    desc = (AugGeom * len(params))()
    for i, p in enumerate(params):
        d = desc[i]
        d.m[:] = [float(v) for v in np.asarray(p["M"], np.float64).reshape(-1)[:9]]
        d.perspective, d.mosaic, d.flip = int(p["perspective"]), int(p["mosaic"]), int(p["flip"])
        d.src[:] = [int(v) for v in p["src"]]
        d.xc, d.yc = int(p.get("xc", 0)), int(p.get("yc", 0))
    return desc


def augment_geometric(imgs, params, out=None):
    """YOLOv5's geometric augmentation on a CUDA uint8 [N, 3, H, W] planar BGR batch (yfv2_aug_geometric): per output image,
    load_mosaic's canvas (or the image src[0] alone), cv2.warpAffine / cv2.warpPerspective of it by M with borderValue 114, then
    np.fliplr.  params: N dicts (utils.device_aug.draw_geometric returns them) with M (3x3, canvas -> output, as cv2 receives it),
    perspective, mosaic, src (4 batch indices; src[0] alone without mosaic), xc, yc and flip.  Returns a new tensor, or writes
    `out`, which must not overlap `imgs`."""
    _require_cuda(imgs, "imgs")
    if imgs.dtype != torch.uint8 or imgs.dim() != 4 or imgs.shape[1] != 3:
        raise TypeError("augment_geometric expects uint8 [N, 3, H, W] images")
    imgs = imgs.contiguous()
    N, _, H, W = imgs.shape
    if len(params) != N:
        raise ValueError("one geometric descriptor per image")
    desc = geom_descriptors(params)
    if out is None:
        out = torch.empty_like(imgs)
    elif out.dtype != torch.uint8 or tuple(out.shape) != tuple(imgs.shape) or not out.is_contiguous() or out.device != imgs.device:
        raise ValueError("out must be a contiguous uint8 tensor of the batch's shape on its device")
    with torch.cuda.device(imgs.device):
        _check(lib().yfv2_aug_geometric(ctypes.c_void_p(imgs.data_ptr()), ctypes.c_void_p(out.data_ptr()), N, H, W, desc,
                                        _stream(imgs.device)), "aug_geometric")
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


def resize_bgr(frames, W, H, device=None, out=None):
    """cv2.resize(frame, (W, H), interpolation=cv2.INTER_LINEAR) of every frame, transposed to the [N, 3, H, W] uint8 batch the
    network takes (test.py:34-37), bit for bit, in one kernel.  frames: HWC uint8 BGR numpy arrays or CUDA tensors, any sizes
    (host arrays are copied to `device` first; a CUDA tensor that is a row crop of a larger frame is read in place)."""
    return _resize("resize_bgr", frames, "bgr", ("bgr",), W, H, device, out)


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
        device = _device("decode_jpeg", (), device)
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
        [N, 3, H, W] tensor on the batch's device; None: a new one), returned, on the current stream without synchronising; the
        flags as decode() sets them."""
        out = _out("decode_resize_jpeg", out, len(self.infos), H, W, self.device)
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
    out = b.decode_resize(out, W, H)
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


def _uint8_plane(p, what, fn):
    """p as a uint8 2-D torch tensor; a host numpy array is wrapped, not copied."""
    if not isinstance(p, torch.Tensor):
        p = np.asarray(p)
        if p.dtype != np.uint8 or p.ndim != 2:
            raise Yfv2Error("%s: %s must be a uint8 2-D array, got %s %s" % (fn, what, p.dtype, p.shape))
        p = torch.from_numpy(p if min(p.strides, default=0) >= 0 else np.ascontiguousarray(p))
    elif p.dtype != torch.uint8 or p.dim() != 2:
        raise Yfv2Error("%s: %s must be a uint8 2-D tensor, got %s %s" % (fn, what, p.dtype, tuple(p.shape)))
    return p


def _yuv420_planes(f, layout, i, fn):
    """Frame i as uint8 2-D planes, checked, not copied: (y, uv) for NV12 / NV21, (y, u, v) for I420 / YV12.  A single buffer is
    cv2's [h*3/2, w] layout: the luma rows, then the chroma (interleaved rows for NV12 / NV21; for I420 / YV12 the two w/2-wide
    planes back to back, read from a contiguous buffer)."""
    interleaved = layout in ("nv12", "nv21")
    if isinstance(f, (tuple, list)):
        planes = tuple(_uint8_plane(p, "frame %d plane %d" % (i, k), fn) for k, p in enumerate(f))
        if len(planes) != (2 if interleaved else 3):
            raise Yfv2Error("%s: frame %d: %s takes %s, got %d planes"
                            % (fn, i, layout, "(y, uv)" if interleaved else "(y, u, v)", len(planes)))
        y = planes[0]
        h, w = y.shape
        chroma = [(h // 2, w)] if interleaved else [(h // 2, w // 2)] * 2
        for k, (p, want) in enumerate(zip(planes[1:], chroma)):
            if tuple(p.shape) != want or h % 2 or w % 2:
                raise Yfv2Error("%s: frame %d: y %s needs even sizes and chroma planes of %s, plane %d is %s"
                                % (fn, i, tuple(y.shape), want, k + 1, tuple(p.shape)))
        return planes
    buf = _uint8_plane(f, "frame %d" % i, fn)
    rows, w = buf.shape
    h = rows // 3 * 2
    if rows % 3 or h <= 0 or w <= 0 or w % 2:
        raise Yfv2Error("%s: frame %d: a single buffer is [h*3/2, w] with h, w even and > 0, got %s" % (fn, i, tuple(buf.shape)))
    if interleaved:
        return buf[:h], buf[h:]
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
    return _resize("resize_yuv420", frames, layout, YUV420_LAYOUTS, W, H, device, out)


# Layouts yfv2_resize_strided_u8 takes: the byte offsets of B, G, R within a pixel of each packed one.  "rgb_chw" ([3, h, w], R
# plane first) is built from its channel stride instead.
STRIDED_LAYOUTS = ("rgb", "bgra", "rgba", "gray", "rgb_chw")
_BGR_OFFSETS = {"rgb": (2, 1, 0), "bgra": (0, 1, 2), "rgba": (2, 1, 0), "gray": (0, 0, 0)}
# packed YUV 4:2:2 (yfv2_resize_yuv422_u8): the byte offsets of the first Y, of U and of V within a 4-byte macropixel
YUV422_LAYOUTS = ("yuyv", "uyvy", "yvyu")
_YUV422_OFFSETS = {"yuyv": (0, 1, 3), "uyvy": (1, 0, 2), "yvyu": (0, 3, 1)}
# bytes per pixel of each packed layout
_CHANNELS = {"bgr": 3, "rgb": 3, "bgra": 4, "rgba": 4, "gray": 1, "yuyv": 2, "uyvy": 2, "yvyu": 2}
LAYOUTS = ("bgr",) + YUV420_LAYOUTS + STRIDED_LAYOUTS + YUV422_LAYOUTS
# raw Bayer frames (yfv2_resize_bayer_u8): "bayer_<xy>" is cv2's COLOR_Bayer<XY>2BGR, "bayer_<xy>_ea" its edge-aware
# COLOR_Bayer<XY>2BGR_EA; _BAYER_RED holds the column and row parity of the red sites of each pattern
_BAYER_RED = {"bg": (0, 0), "gb": (1, 0), "rg": (1, 1), "gr": (0, 1)}
BAYER_LAYOUTS = tuple("bayer_" + k for k in _BAYER_RED) + tuple("bayer_%s_ea" % k for k in _BAYER_RED)
_FRAME_LAYOUTS = LAYOUTS + BAYER_LAYOUTS          # every layout resize_frames, encode_jpeg and crop_frame take
# the descriptor kind (yfv2_jpeg_enc_src.kind) of each layout, and the union member of yfv2_jpeg_enc_src.f each kind fills: the
# resize entry yfv2_resize_<member>_u8 takes an array of it
_KIND = dict([("bgr", JPEG_SRC_BGR), ("gray", JPEG_SRC_GRAY)] + [(k, JPEG_SRC_YUV420) for k in YUV420_LAYOUTS]
             + [(k, JPEG_SRC_STRIDED) for k in STRIDED_LAYOUTS if k != "gray"] + [(k, JPEG_SRC_YUV422) for k in YUV422_LAYOUTS]
             + [(k, JPEG_SRC_BAYER) for k in BAYER_LAYOUTS])
_MEMBER = ("bgr", "strided", "strided", "yuv420", "yuv422", "bayer")
_DESC = dict(_EncFrame._fields_ + [("remap", RemapFrame), ("warp", WarpFrame)])


class BayerWindow:
    """The w x h window at (x0, y0) of cv2.cvtColor(raw, COLOR_Bayer??2BGR) of a whole raw Bayer frame: what crop_frame returns for
    the Bayer layouts, and what resize_frames, encode_jpeg, frame_size and crop_frame take for them besides whole frames.  raw is
    the whole [fh, fw] uint8 frame (numpy or CUDA), never copied.  The demosaic of a pixel reads its neighbours and the frame's
    edges, so the window cannot be a crop of the raw bytes."""
    __slots__ = ("raw", "x0", "y0", "w", "h")

    def __init__(self, raw, x0, y0, w, h):
        self.raw, self.x0, self.y0, self.w, self.h = raw, int(x0), int(y0), int(w), int(h)

    def __repr__(self):
        return "BayerWindow(raw %s, x0 %d, y0 %d, %dx%d)" % (tuple(self.raw.shape), self.x0, self.y0, self.w, self.h)


REMAP_MAX_SIDE = 32766          # cv2.remap asserts map sides below SHRT_MAX


def convert_maps(mx, my):
    """cv2.convertMaps(mx, my, cv2.CV_16SC2) of float32 maps (torch tensors of one shape, on any device): (xy int16 [h, w, 2],
    code int16 [h, w] holding cv2's uint16 map2).  X = rint_half_even(fl32(x * 32)), or INT32_MIN for NaN, +-inf and |x * 32| >=
    2^31 (x86's cvRound); x0 = saturate_int16(X >> 5), j = X & 31; the same for y; code = 32 i + j.  The non-finite and huge
    entries are masked before any float -> int cast, whose result for them differs between the CPU and the device."""
    def fixed(v):
        v = v * 32.0                                          # fp32, exact unless it overflows to inf (masked)
        ok = torch.isfinite(v) & (v.abs() < 2.0 ** 31)
        r = torch.round(torch.where(ok, v, torch.zeros_like(v))).to(torch.int64)     # half to even, as cvRound
        r = torch.where(ok, r, torch.full_like(r, -2 ** 31))
        return (r >> 5).clamp(-32768, 32767), r & 31
    x0, j = fixed(mx)
    y0, i = fixed(my)
    return torch.stack([x0, y0], -1).to(torch.int16), (32 * i + j).to(torch.int16)


def _map_tensor(m, what):
    """A map plane as a torch tensor (numpy wrapped, not copied; uint16 viewed as int16) and whether it was unsigned."""
    if isinstance(m, torch.Tensor):
        if m.dtype == torch.uint16:
            return m.view(torch.int16), True
        return m, False
    m = np.asarray(m)
    if m.dtype == np.uint16:
        return torch.from_numpy(np.ascontiguousarray(m).view(np.int16)), True
    if m.dtype not in (np.float32, np.int16):
        raise Yfv2Error("RemapMaps: %s must be float32, int16 or uint16 (cv2's map types), got %s" % (what, m.dtype))
    return torch.from_numpy(m if min(m.strides, default=0) >= 0 else np.ascontiguousarray(m)), False


class RemapMaps:
    """cv2.remap's maps, held on a CUDA device in cv2's fixed form: xy int16 [mh, mw, 2] (CV_16SC2 map1) and code int16 [mh, mw]
    (CV_16UC1 map2's bits), both contiguous.  Takes what cv2.remap takes for INTER_LINEAR, as numpy arrays or torch tensors:
      float maps   map1, map2 float32 [h, w] (x and y), or map1 float32 [h, w, 2] with map2 None: converted once exactly as
                   cv2.convertMaps(map1, map2, CV_16SC2) (convert_maps), so the remap gives cv2.remap's bytes for them;
      fixed maps   map1 int16 [h, w, 2] and map2 uint16 (or int16) [h, w], what cv2.convertMaps or
                   cv2.initUndistortRectifyMap(..., CV_16SC2) return: taken as they are (only map2's low 10 bits are read).
    A fixed map and the conversion of the float map it was made from may differ (initUndistortRectifyMap rounds in fp64), so
    pass the form whose cv2.remap bytes you want.  h, w in 1..32766, as cv2 requires.  device: where the maps are held (default:
    map1's CUDA device, else the current one)."""
    __slots__ = ("xy", "code", "mw", "mh")

    def __init__(self, map1, map2=None, device=None):
        m1, u1 = _map_tensor(map1, "map1")
        m2, u2 = (None, False) if map2 is None else _map_tensor(map2, "map2")
        if m1.dtype == torch.float32:
            if m2 is None:
                if m1.dim() != 3 or m1.shape[2] != 2:
                    raise Yfv2Error("RemapMaps: a single float map must be float32 [h, w, 2], got %s" % (tuple(m1.shape),))
                mx, my = m1[..., 0], m1[..., 1]
            else:
                if m2.dtype != torch.float32 or m1.dim() != 2 or tuple(m2.shape) != tuple(m1.shape):
                    raise Yfv2Error("RemapMaps: float maps must be two float32 [h, w] planes of one shape, got %s %s and %s %s"
                                    % (m1.dtype, tuple(m1.shape), m2.dtype, tuple(m2.shape)))
                mx, my = m1, m2
            xy, code = convert_maps(mx, my)
        elif m1.dtype == torch.int16 and not u1:
            if m1.dim() != 3 or m1.shape[2] != 2:
                raise Yfv2Error("RemapMaps: a fixed map1 must be int16 [h, w, 2], got %s" % (tuple(m1.shape),))
            if m2 is None or m2.dtype != torch.int16 or tuple(m2.shape) != tuple(m1.shape[:2]):
                raise Yfv2Error("RemapMaps: a fixed map1 needs map2 uint16 [h, w] (its interpolation codes), got %s"
                                % ("None" if m2 is None else "%s %s" % ("uint16" if u2 else m2.dtype, tuple(m2.shape))))
            xy, code = m1, m2
        else:
            raise Yfv2Error("RemapMaps: map1 must be float32 or int16 (cv2's map types), got %s" % ("uint16" if u1 else m1.dtype))
        mh, mw = xy.shape[:2]
        if not (1 <= mw <= REMAP_MAX_SIDE and 1 <= mh <= REMAP_MAX_SIDE):
            raise Yfv2Error("RemapMaps: map sides must be in 1..%d, got %dx%d" % (REMAP_MAX_SIDE, mw, mh))
        if device is None:
            device = m1.device if m1.is_cuda else torch.device("cuda", torch.cuda.current_device())
        device = torch.device(device)
        if device.type != "cuda":
            raise Yfv2Error("RemapMaps: maps are held on a CUDA device (no CPU fallback), got %s" % device)
        self.xy, self.code = xy.to(device).contiguous(), code.to(device).contiguous()
        self.mw, self.mh = int(mw), int(mh)

    def __repr__(self):
        return "RemapMaps(%dx%d on %s)" % (self.mw, self.mh, self.xy.device)


class RemapView:
    """The w x h window at (x0, y0) of cv2.remap(cv2.cvtColor(frame, COLOR_<LAYOUT>2BGR), map1, map2, cv2.INTER_LINEAR) (constant 0
    border): a lens-corrected view of a frame, read where it is used, never stored.  frame: any frame resize_frames takes for the
    layout (a BayerWindow or a crop included: the maps address its converted pixels); maps: a RemapMaps.  The layout passed with
    a view names its frame's layout.  The window defaults to the whole remapped image (the map's size).  resize_frames,
    remap_frames, encode_jpeg, crop_frame, frame_size and the detection and tracking helpers take views; boxes come back in the
    view's pixels."""
    __slots__ = ("frame", "maps", "x0", "y0", "w", "h")

    def __init__(self, frame, maps, x0=0, y0=0, w=None, h=None):
        if not isinstance(maps, RemapMaps):
            raise Yfv2Error("RemapView: maps must be a RemapMaps, got %s" % type(maps).__name__)
        self.frame, self.maps, self.x0, self.y0 = frame, maps, int(x0), int(y0)
        self.w = maps.mw - self.x0 if w is None else int(w)
        self.h = maps.mh - self.y0 if h is None else int(h)

    def __repr__(self):
        return "RemapView(%r, %r, x0 %d, y0 %d, %dx%d)" % (type(self.frame).__name__, self.maps, self.x0, self.y0, self.w, self.h)


WARP_MAX_SIDE = 32767


def _warp_desc(m, perspective, inverse, dsize, x0=0, y0=0, w=1, h=1):
    """A WarpFrame of the matrix, output size and window, its inner frame left empty."""
    d = WarpFrame(0, x0, y0, w, h)
    d.m[:] = list(m) + [0.0] * (9 - len(m))
    d.perspective, d.inverse, (d.dw, d.dh) = int(perspective), int(inverse), dsize
    return d


def warp_matrix(M, inverse=False):
    """The destination -> source matrix (float64 [3, 3]) cv2.warpAffine (M 2x3) or cv2.warpPerspective (M 3x3) samples with: M
    itself with inverse (WARP_INVERSE_MAP), else M inverted on the host as cv2 inverts it, bit for bit (yfv2_warp_matrix).  Raises
    Yfv2Error for what a WarpView of M refuses (a singular M, non-finite entries)."""
    m, perspective = _warp_entries(M, "warp_matrix")
    out = (ctypes.c_double * 9)()
    d = _warp_desc(m, perspective, inverse, (1, 1))
    if lib().yfv2_warp_matrix(ctypes.byref(d), out):
        raise Yfv2Error(lib().yfv2_last_error().decode())
    return np.array(list(out), np.float64).reshape(3, 3)


def _warp_entries(M, fn):
    """M (a 2x3 or 3x3 numpy array or nested list) as a tuple of its float64 values, and whether it is 3x3."""
    try:
        a = np.array(M, dtype=np.float64)
    except (TypeError, ValueError):
        raise Yfv2Error("%s: M must be a 2x3 or 3x3 matrix of numbers, got %r" % (fn, type(M).__name__))
    if a.shape not in ((2, 3), (3, 3)):
        raise Yfv2Error("%s: M must be 2x3 (warpAffine) or 3x3 (warpPerspective), got shape %s" % (fn, a.shape))
    return tuple(float(v) for v in a.reshape(-1)), a.shape == (3, 3)


class WarpView:
    """The w x h window at (x0, y0) of cv2.warpAffine(img, M, dsize) (M 2x3) or cv2.warpPerspective(img, M, dsize) (M 3x3, whatever
    its last row), img = cv2.cvtColor(frame, COLOR_<LAYOUT>2BGR), INTER_LINEAR with the constant 0 border, and cv2.WARP_INVERSE_MAP
    when inverse: a rotated, de-skewed or bird's-eye view of a frame, computed where it is read, never stored.  frame: any frame
    resize_frames takes for the layout (a BayerWindow or a crop included: M addresses its converted pixels); M: numpy or nested
    lists, copied as float64 (later changes to the caller's array do not reach the view); dsize: (width, height), as cv2 takes it,
    each in 1..32767.  The window defaults to the whole warped image.  The layout passed with a view names its frame's layout.
    resize_frames, warp_frames, encode_jpeg, crop_frame, frame_size and the detection and tracking helpers take views; boxes come
    back in the view's pixels."""
    __slots__ = ("frame", "m", "perspective", "inverse", "dw", "dh", "x0", "y0", "w", "h")

    def __init__(self, frame, M, dsize, x0=0, y0=0, w=None, h=None, inverse=False):
        self.m, self.perspective = _warp_entries(M, "WarpView")
        if len(dsize) != 2:
            raise Yfv2Error("WarpView: dsize must be (width, height), got %r" % (dsize,))
        self.frame, self.inverse = frame, bool(inverse)
        self.dw, self.dh = int(dsize[0]), int(dsize[1])
        self.x0, self.y0 = int(x0), int(y0)
        self.w = self.dw - self.x0 if w is None else int(w)
        self.h = self.dh - self.y0 if h is None else int(h)

    def over(self, frame, x0, y0, w, h):
        """The same warp of `frame` (checked or placed elsewhere), with the window (x0, y0, w, h)."""
        v = object.__new__(WarpView)
        for k in self.__slots__:
            setattr(v, k, getattr(self, k))
        v.frame, v.x0, v.y0, v.w, v.h = frame, x0, y0, w, h
        return v

    def __repr__(self):
        return "WarpView(%r, %s, %dx%d output, x0 %d, y0 %d, %dx%d%s)" % (
            type(self.frame).__name__, "perspective" if self.perspective else "affine", self.dw, self.dh, self.x0, self.y0,
            self.w, self.h, ", inverse" if self.inverse else "")


def frame_size(frame, layout):
    """(h, w) in pixels of a frame in the given layout, as resize_frames takes it (of its window for a BayerWindow, a RemapView or
    a WarpView)."""
    if isinstance(frame, (BayerWindow, RemapView, WarpView)):
        return frame.h, frame.w
    if layout in YUV420_LAYOUTS:
        if isinstance(frame, (tuple, list)):
            return tuple(frame[0].shape[:2])
        return frame.shape[0] // 3 * 2, frame.shape[1]
    return tuple(frame.shape[1:3]) if layout == "rgb_chw" else tuple(frame.shape[:2])


def _layout_frame(f, layout, i, fn):
    """Frame i of a strided or 4:2:2 layout as a uint8 tensor of the layout's shape, checked, not copied."""
    shape = ("[3, h, w]" if layout == "rgb_chw" else "[h, w]" if layout == "gray" else "[h, w, %d]" % _CHANNELS[layout])
    if not isinstance(f, torch.Tensor):
        f = np.asarray(f)
        if f.dtype != np.uint8:
            raise Yfv2Error("%s: frame %d (%s) must be uint8 %s, got %s %s" % (fn, i, layout, shape, f.dtype, f.shape))
        f = torch.from_numpy(f if min(f.strides, default=0) >= 0 else np.ascontiguousarray(f))
    ok = f.dtype == torch.uint8 and f.dim() == (2 if layout == "gray" else 3) and f.numel() > 0
    if ok and layout == "rgb_chw":
        ok = f.shape[0] == 3
    elif ok and layout != "gray":
        ok = f.shape[2] == _CHANNELS[layout]
    if not ok:
        raise Yfv2Error("%s: frame %d (%s) must be uint8 %s with h, w > 0, got %s %s"
                        % (fn, i, layout, shape, f.dtype, tuple(f.shape)))
    if layout in YUV422_LAYOUTS and f.shape[1] % 2:
        raise Yfv2Error("%s: frame %d (%s): 4:2:2 needs an even width (two pixels per macropixel), got w = %d"
                        % (fn, i, layout, f.shape[1]))
    return f


def _bayer_window(f, layout, i, fn):
    """Frame i of a Bayer layout, a whole [fh, fw] uint8 frame or a BayerWindow, as a BayerWindow over a uint8 2-D tensor, checked,
    not copied."""
    win = f if isinstance(f, BayerWindow) else None
    raw = _uint8_plane(win.raw if win else f, "frame %d (%s)" % (i, layout), fn)
    fh, fw = raw.shape
    if fh < 1 or fw < 1:
        raise Yfv2Error("%s: frame %d (%s) must be uint8 [h, w] with h, w > 0, got %s" % (fn, i, layout, tuple(raw.shape)))
    if win is None:
        return BayerWindow(raw, 0, 0, fw, fh)
    if win.w < 1 or win.h < 1 or win.x0 < 0 or win.y0 < 0 or win.x0 + win.w > fw or win.y0 + win.h > fh:
        raise Yfv2Error("%s: frame %d (%s): window (x0 %d, y0 %d, %dx%d) is not inside the %dx%d frame"
                        % (fn, i, layout, win.x0, win.y0, win.w, win.h, fw, fh))
    return BayerWindow(raw, win.x0, win.y0, win.w, win.h)


def _check_frame(f, layout, i, fn):
    """Checks frame i against its layout without copying or launching anything; returns what _describe takes: the BGR array or
    tensor, the planes of a 4:2:0 frame, a BayerWindow over a tensor for Bayer, a uint8 tensor of the layout's shape for the
    others, a RemapView or WarpView over the checked frame for a view.  A refusal names fn, the public function called."""
    if isinstance(f, (RemapView, WarpView)) and isinstance(f.frame, (RemapView, WarpView)):
        raise Yfv2Error("%s: frame %d: a %s of a %s (views do not nest: compose the maps or matrices instead)"
                        % (fn, i, type(f).__name__, type(f.frame).__name__))
    if isinstance(f, WarpView):
        if not (1 <= f.dw <= WARP_MAX_SIDE and 1 <= f.dh <= WARP_MAX_SIDE):
            raise Yfv2Error("%s: frame %d (%s view): dsize %dx%d outside 1..%d" % (fn, i, layout, f.dw, f.dh, WARP_MAX_SIDE))
        if f.w < 1 or f.h < 1 or f.x0 < 0 or f.y0 < 0 or f.x0 + f.w > f.dw or f.y0 + f.h > f.dh:
            raise Yfv2Error("%s: frame %d (%s view): window (x0 %d, y0 %d, %dx%d) is not inside the %dx%d output"
                            % (fn, i, layout, f.x0, f.y0, f.w, f.h, f.dw, f.dh))
        d = _warp_desc(f.m, f.perspective, f.inverse, (f.dw, f.dh))
        if lib().yfv2_warp_matrix(ctypes.byref(d), (ctypes.c_double * 9)()):
            raise Yfv2Error("%s: frame %d (%s view): %s" % (fn, i, layout, lib().yfv2_last_error().decode().split(": ", 1)[1]))
        return f.over(_check_frame(f.frame, layout, i, fn), f.x0, f.y0, f.w, f.h)
    if isinstance(f, RemapView):
        m = f.maps
        if f.w < 1 or f.h < 1 or f.x0 < 0 or f.y0 < 0 or f.x0 + f.w > m.mw or f.y0 + f.h > m.mh:
            raise Yfv2Error("%s: frame %d (%s view): window (x0 %d, y0 %d, %dx%d) is not inside the %dx%d map"
                            % (fn, i, layout, f.x0, f.y0, f.w, f.h, m.mw, m.mh))
        return RemapView(_check_frame(f.frame, layout, i, fn), m, f.x0, f.y0, f.w, f.h)
    kind = _KIND[layout]
    if kind == JPEG_SRC_BAYER:
        return _bayer_window(f, layout, i, fn)
    if kind == JPEG_SRC_BGR:
        if isinstance(f, torch.Tensor):
            ok = f.dtype == torch.uint8
        else:
            f = np.asarray(f)
            ok = f.dtype == np.uint8
        if not ok or f.ndim != 3 or f.shape[2] != 3:
            raise Yfv2Error("%s: frame %d (bgr) must be uint8 [h, w, 3], got %s %s" % (fn, i, f.dtype, tuple(f.shape)))
        return f
    if kind == JPEG_SRC_YUV420:
        return _yuv420_planes(f, layout, i, fn)
    return _layout_frame(f, layout, i, fn)


def _checked_frames(fn, frames, layout, allowed=_FRAME_LAYOUTS):
    """The frames as a list, each checked (_check_frame), and one layout name per frame from `layout` (one name, or one per frame),
    each among `allowed`."""
    frames = list(frames)
    layouts = [layout] * len(frames) if isinstance(layout, str) else list(layout)
    for lay in layouts if layouts else [layout]:
        if not isinstance(lay, str) or lay not in allowed:
            raise Yfv2Error("%s: layout must be one of %s, got %r" % (fn, ", ".join(allowed), lay))
    if not frames:
        raise Yfv2Error("%s: no frames" % fn)
    if len(layouts) != len(frames):
        raise Yfv2Error("%s: %d layouts for %d frames" % (fn, len(layouts), len(frames)))
    return [_check_frame(f, lay, i, fn) for i, (f, lay) in enumerate(zip(frames, layouts))], layouts


def _tensors(f):
    """The arrays or tensors a checked frame reads: its planes, a BayerWindow's raw frame, a RemapView's frame and then its maps, a
    WarpView's frame."""
    if isinstance(f, RemapView):
        return _tensors(f.frame) + (f.maps.xy,)
    if isinstance(f, WarpView):
        return _tensors(f.frame)
    return f if isinstance(f, tuple) else (f.raw,) if isinstance(f, BayerWindow) else (f,)


def _device(fn, frames, device):
    """The CUDA device a call runs on, with its index: `device`, else that of the first CUDA tensor among the checked frames (or
    their planes, or a view's maps), else the current one."""
    if device is None:
        device = next((t.device for f in frames for t in _tensors(f) if isinstance(t, torch.Tensor) and t.is_cuda), None)
    device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    if device.type != "cuda":
        raise Yfv2Error("%s: runs on CUDA devices only (no CPU fallback)" % fn)
    return device if device.index is not None else torch.device("cuda", torch.cuda.current_device())


def _out(fn, out, N, H, W, device):
    """out checked to be a contiguous uint8 [N, 3, H, W] tensor on device, or a new one when None."""
    if out is None:
        return torch.empty((N, 3, H, W), dtype=torch.uint8, device=device)
    if (not isinstance(out, torch.Tensor) or tuple(out.shape) != (N, 3, H, W) or out.dtype != torch.uint8 or not out.is_contiguous()
            or out.device != device):
        raise Yfv2Error("%s: out must be a contiguous uint8 tensor of shape %s on %s" % (fn, (N, 3, H, W), device))
    return out


def _describe(f, layout, device, keep):
    """The descriptor of frame f (as _check_frame returned it) with its pixels on `device`: a JpegEncSrc of the layout's kind, its
    union member filled and the whole frame as its region.  The only code that places frames: host frames are copied to
    `device`; a CUDA frame is read in place when its strides fit the descriptor, else a contiguous copy of it is.  The device
    tensors read go to keep, which must hold them until the launch is queued: a freed block could take the next frame's copy.
    For a RemapView: a RemapFrame of its frame's descriptor (grey as strided), its maps on `device` and its window; for a
    WarpView, a WarpFrame of its frame's descriptor, its matrix, output size and window."""
    if isinstance(f, WarpView):
        s = _describe(f.frame, layout, device, keep)
        r = _warp_desc(f.m, f.perspective, f.inverse, (f.dw, f.dh), f.x0, f.y0, f.w, f.h)
        r.kind, r.f = JPEG_SRC_STRIDED if s.kind == JPEG_SRC_GRAY else s.kind, s.f
        return r
    if isinstance(f, RemapView):
        s = _describe(f.frame, layout, device, keep)
        r = RemapFrame(JPEG_SRC_STRIDED if s.kind == JPEG_SRC_GRAY else s.kind, f.x0, f.y0, f.w, f.h)
        r.f = s.f
        xy, code = f.maps.xy.to(device), f.maps.code.to(device)
        r.map.xy, r.map.xy_pitch, r.map.code, r.map.code_pitch = xy.data_ptr(), 4 * f.maps.mw, code.data_ptr(), 2 * f.maps.mw
        r.map.mw, r.map.mh = f.maps.mw, f.maps.mh
        keep += [xy, code]
        return r
    kind = _KIND[layout]
    s = JpegEncSrc(kind)
    if kind == JPEG_SRC_BAYER:                                # the whole raw frame, any row stride, unit column stride
        raw = f.raw.to(device)
        fh, fw = raw.shape
        if (fw > 1 and raw.stride(1) != 1) or (fh > 1 and raw.stride(0) < fw):
            raw = raw.contiguous()
        e = s.f.bayer
        # torch keeps any stride on a dimension of size 1 (contiguous() too); one row has no next row, so its pitch is fw
        e.data, e.pitch, e.fh, e.fw = raw.data_ptr(), raw.stride(0) if fh > 1 else fw, fh, fw
        e.x0, e.y0, e.w, e.h = f.x0, f.y0, f.w, f.h
        e.red_x, e.red_y = _BAYER_RED[layout[6:8]]
        e.edge_aware = layout.endswith("_ea")
        s.w, s.h = f.w, f.h
        keep.append(raw)
        return s
    if kind == JPEG_SRC_YUV420:
        planes = [p.to(device) for p in f]
        planes = [p if p.stride(1) == 1 else p.contiguous() for p in planes]
        y, u, e = planes[0], planes[1], s.f.yuv420
        if len(planes) == 2:                                  # NV12 / NV21: one interleaved chroma plane, U first for NV12
            e.u, e.v, e.uv_pitch, e.uv_step = u.data_ptr() + (layout == "nv21"), u.data_ptr() + (layout == "nv12"), u.stride(0), 2
        else:
            v = planes[2]
            if u.stride(0) != v.stride(0):                    # one chroma pitch per descriptor
                planes[1:] = u, v = u.contiguous(), v.contiguous()
            e.u, e.v, e.uv_pitch, e.uv_step = u.data_ptr(), v.data_ptr(), u.stride(0), 1
        e.y, e.y_pitch = y.data_ptr(), y.stride(0)
        e.h, e.w = s.h, s.w = y.shape
        keep += planes
        return s
    if not isinstance(f, torch.Tensor):                       # a host BGR array: the other layouts' checks return tensors
        f = torch.from_numpy(np.ascontiguousarray(f))
    f = f.to(device)
    st = f.stride()
    if layout == "rgb_chw":                                   # any channel and row stride, unit column stride
        _, h, w = f.shape
        if st[2] != 1 or st[1] < w:
            f = f.contiguous()
            st = f.stride()
        p = f.data_ptr()
        e = s.f.strided
        e.b, e.g, e.r, e.pitch, e.step = p + 2 * st[0], p + st[0], p, st[1], 1
    else:                                                     # packed: pixels `step` bytes apart, rows at least w pixels apart
        (h, w), step = f.shape[:2], _CHANNELS[layout]
        if st[1] != step or (layout != "gray" and st[2] != 1) or st[0] < step * w:
            f = f.contiguous()
            st = f.stride()
        p = f.data_ptr()
        if kind == JPEG_SRC_BGR:
            e = s.f.bgr
            e.data = p
        elif kind == JPEG_SRC_YUV422:
            e = s.f.yuv422
            e.y, e.u, e.v = (p + o for o in _YUV422_OFFSETS[layout])
        else:
            e = s.f.strided
            e.b, e.g, e.r = (p + o for o in _BGR_OFFSETS[layout])
            e.step = step
        e.pitch = st[0]
    e.h, e.w = s.h, s.w = h, w
    keep.append(f)
    return s


def _resize(fn, frames, layout, allowed, W, H, device, out):
    """resize_bgr, resize_yuv420 and resize_frames: every frame checked, then one yfv2_resize_<member>_u8 call for each run of
    consecutive frames that fill the same descriptor (RemapViews of any kind: yfv2_resize_remap_u8; WarpViews:
    yfv2_resize_warp_u8), each into its slice of out."""
    checked, layouts = _checked_frames(fn, frames, layout, allowed)
    device = _device(fn, checked, device)
    N = len(checked)
    out = _out(fn, out, N, H, W, device)

    def member_of(k):
        f = checked[k]
        return "remap" if isinstance(f, RemapView) else "warp" if isinstance(f, WarpView) else _MEMBER[_KIND[layouts[k]]]

    i = 0
    while i < N:
        member, j = member_of(i), i + 1
        while j < N and member_of(j) == member:
            j += 1
        keep, desc = [], _DESC[member]
        lo, hi = JpegEncSrc.f.offset, JpegEncSrc.f.offset + ctypes.sizeof(desc)     # the member's bytes in a JpegEncSrc
        if member in ("remap", "warp"):
            lo, hi = 0, ctypes.sizeof(desc)
        srcs = [bytes(_describe(checked[k], layouts[k], device, keep)) for k in range(i, j)]
        descs = (desc * (j - i)).from_buffer_copy(b"".join(src[lo:hi] for src in srcs))
        entry = getattr(lib(), "yfv2_resize_%s_u8" % member)
        with torch.cuda.device(device):
            _check(entry(descs, j - i, H, W, ctypes.c_void_p(out[i].data_ptr()), _stream(device)), "resize_%s_u8" % member)
        i = j
    return out


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
      "bayer_bg" | "bayer_gb"           [h, w] raw Bayer (BAYER_LAYOUTS), COLOR_Bayer<XY>2BGR; "bayer_<xy>_ea": _EA, the
        | "bayer_rg" | "bayer_gr"       edge-aware demosaic; or a BayerWindow of one (crop_frame)
    and a RemapView of a frame of any of these layouts (layout: its frame's): cv2.remap(INTER_LINEAR) of the converted frame,
    cropped to the view's window, computed where the resize reads it (yfv2_resize_remap_u8); a WarpView likewise with
    cv2.warpAffine / cv2.warpPerspective (yfv2_resize_warp_u8).
    Frames are numpy arrays or CUDA tensors; CUDA views with larger row strides or crop offsets are read in place (for
    "rgb_chw" any channel and row stride with unit column stride), host arrays are copied to `device`.  Consecutive frames of
    one descriptor kind go to one call (yfv2_resize_bgr_u8 / _yuv420_u8 / _strided_u8 / _yuv422_u8 / _bayer_u8 / _remap_u8 /
    _warp_u8), each
    into its slice of `out`.  Every frame is checked before anything is copied or launched."""
    return _resize("resize_frames", frames, layout, _FRAME_LAYOUTS, W, H, device, out)


def remap_frames(views, layout, device=None):
    """cv2.remap(cv2.cvtColor(frame, COLOR_<LAYOUT>2BGR), map1, map2, cv2.INTER_LINEAR)[y0:y0+h, x0:x0+w] of every RemapView, bit
    for bit, computed on the device (yfv2_remap_u8): a list of CUDA uint8 [h, w, 3] BGR tensors.  layout: the views' frames'
    layout, one name or one per view.  Every view is checked before anything is copied or launched."""
    return _view_frames("remap_frames", RemapView, views, layout, device)


def warp_frames(views, layout, device=None):
    """cv2.warpAffine / cv2.warpPerspective(cv2.cvtColor(frame, COLOR_<LAYOUT>2BGR), M, dsize, INTER_LINEAR)[y0:y0+h, x0:x0+w] of
    every WarpView, bit for bit, computed on the device (yfv2_warp_u8): a list of CUDA uint8 [h, w, 3] BGR tensors.  layout: the
    views' frames' layout, one name or one per view.  Every view is checked before anything is copied or launched."""
    return _view_frames("warp_frames", WarpView, views, layout, device)


def _view_frames(fn, cls, views, layout, device):
    """remap_frames and warp_frames: every view of class cls checked, then one yfv2_remap_u8 / yfv2_warp_u8 call."""
    checked, layouts = _checked_frames(fn, views, layout)
    for i, v in enumerate(checked):
        if not isinstance(v, cls):
            raise Yfv2Error("%s: frame %d is a %s, not a %s" % (fn, i, type(views[i]).__name__, cls.__name__))
    device = _device(fn, checked, device)
    outs = [torch.empty((v.h, v.w, 3), dtype=torch.uint8, device=device) for v in checked]
    keep = []
    member = "remap" if cls is RemapView else "warp"
    descs = (_DESC[member] * len(checked))(*[_describe(v, lay, device, keep) for v, lay in zip(checked, layouts)])
    dst = (ctypes.c_void_p * len(outs))(*[o.data_ptr() for o in outs])
    with torch.cuda.device(device):
        _check(getattr(lib(), "yfv2_%s_u8" % member)(descs, len(checked), dst, _stream(device)), "%s_u8" % member)
    return outs


# cv2's IMWRITE_* ids and IMWRITE_JPEG_SAMPLING_FACTOR_* values (yfv2_jpeg_encode_plan reads the same pairs)
IMWRITE_JPEG_QUALITY, IMWRITE_JPEG_PROGRESSIVE, IMWRITE_JPEG_OPTIMIZE, IMWRITE_JPEG_RST_INTERVAL = 1, 2, 3, 4
IMWRITE_JPEG_LUMA_QUALITY, IMWRITE_JPEG_CHROMA_QUALITY, IMWRITE_JPEG_SAMPLING_FACTOR = 5, 6, 7
JPEG_SAMPLING = {"420": 0x221111, "422": 0x211111, "444": 0x111111, "440": 0x121111, "411": 0x411111}


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
    frame; for a BayerWindow, from its window).  quality (any int, clamped to 0..100 as cv2 does), sampling ("420", "422",
    "444") and restart_interval (MCUs, 0: none) are one value or one per output; params: extra cv2 (IMWRITE_*, value) pairs for
    every output, or a list of them per output.  Everything is checked before anything is launched; a refusal raises Yfv2Error
    naming the output.  Returns a list of bytes, or with device_out=True (arena, offsets, lengths): the uint8 CUDA arena, output i at offsets[i] (host int64 numpy) and
    lengths[i] bytes long (CUDA int64), with no copy to the host."""
    checked, layouts = _checked_frames("encode_jpeg", frames, layout)
    if regions is None:
        regions = [(i, 0, 0, None, None) for i in range(len(checked))]
    regions = [tuple(r) for r in regions]
    n = len(regions)
    if n == 0:
        raise Yfv2Error("encode_jpeg: no regions")
    for k, r in enumerate(regions):
        if len(r) != 5 or not 0 <= int(r[0]) < len(checked):
            raise Yfv2Error("encode_jpeg: region %d must be (frame index in [0, %d), x0, y0, w, h), got %r" % (k, len(checked), r))
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
    device = _device("encode_jpeg", checked, device)
    # each RemapView or WarpView an output reads: computed once (remap_frames, warp_frames) and encoded as the BGR frame it gives
    views = sorted({int(r[0]) for r in regions if isinstance(checked[int(r[0])], (RemapView, WarpView))})
    for k, r in enumerate(regions):
        v = checked[int(r[0])]
        if isinstance(v, (RemapView, WarpView)) and None not in r[3:]:
            x0, y0, w, h = (int(a) for a in r[1:])
            if w < 1 or h < 1 or x0 < 0 or y0 < 0 or x0 + w > v.w or y0 + h > v.h:
                raise Yfv2Error("encode_jpeg: output %d: region (x0 %d, y0 %d, %dx%d) is not inside the %dx%d view"
                                % (k, x0, y0, w, h, v.w, v.h))
    for cls, fn in ((RemapView, remap_frames), (WarpView, warp_frames)):
        idx = [i for i in views if isinstance(checked[i], cls)]
        if idx:
            for i, t in zip(idx, fn([checked[i] for i in idx], [layouts[i] for i in idx], device)):
                checked[i], layouts[i] = t, "bgr"
    srcs = (JpegEncSrc * n)()
    keep, cparams, frame_src = [], [], {}
    for k, r in enumerate(regions):
        i = int(r[0])
        if i not in frame_src:
            frame_src[i] = _describe(checked[i], layouts[i], device, keep)
        srcs[k] = frame_src[i]
        d = srcs[k]
        d.x0, d.y0 = int(r[1]), int(r[2])
        d.w, d.h = d.w if r[3] is None else int(r[3]), d.h if r[4] is None else int(r[4])
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
    that the 2x2 chroma blocks of the crop are those of the frame.  Packed 4:2:2 needs even x0 and w (whole macropixels).  A Bayer
    frame, or a BayerWindow of one, becomes a BayerWindow of the whole raw frame (any offsets): the conversion of a pixel reads its
    neighbours and the frame's edges, so the raw bytes are not cropped.  A RemapView (WarpView) becomes the RemapView (WarpView)
    of the window of its remapped (warped) image (any offsets, whatever its frame's layout).  A crop of a crop is the crop of the
    frame."""
    if layout not in _FRAME_LAYOUTS:
        raise Yfv2Error("crop_frame: layout must be one of %s, got %r" % (", ".join(_FRAME_LAYOUTS), layout))
    f = _check_frame(frame, layout, 0, "crop_frame")
    fh, fw = frame_size(f, layout)
    x0, y0, w, h = int(x0), int(y0), int(w), int(h)
    if w < 1 or h < 1 or x0 < 0 or y0 < 0 or x0 + w > fw or y0 + h > fh:
        raise Yfv2Error("crop_frame: window (x0 %d, y0 %d, %dx%d) is not inside the %dx%d frame" % (x0, y0, w, h, fw, fh))
    if isinstance(f, RemapView):                              # a window of the remapped image: any offsets, any layout
        return RemapView(f.frame, f.maps, f.x0 + x0, f.y0 + y0, w, h)
    if isinstance(f, WarpView):                               # a window of the warped image: any offsets, any layout
        return f.over(f.frame, f.x0 + x0, f.y0 + y0, w, h)
    if layout in YUV420_LAYOUTS and (x0 | y0 | w | h) & 1:
        raise Yfv2Error("crop_frame: %s crops need even x0, y0, w and h (2x2 chroma blocks), got (x0 %d, y0 %d, %dx%d)"
                        % (layout, x0, y0, w, h))
    if layout in YUV422_LAYOUTS and (x0 | w) & 1:
        raise Yfv2Error("crop_frame: %s crops need even x0 and w (two pixels per macropixel), got x0 %d, w %d" % (layout, x0, w))
    if layout in YUV420_LAYOUTS:
        cy = slice(y0 // 2, (y0 + h) // 2)
        if len(f) == 2:                                       # (y, uv)
            return f[0][y0:y0 + h, x0:x0 + w], f[1][cy, x0:x0 + w]
        cx = slice(x0 // 2, (x0 + w) // 2)
        return f[0][y0:y0 + h, x0:x0 + w], f[1][cy, cx], f[2][cy, cx]
    if layout in BAYER_LAYOUTS:
        return BayerWindow(f.raw, f.x0 + x0, f.y0 + y0, w, h)
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

"""CPU restatement of the reference post-process: anchor-grid decode + per-image NMS.

decode()  <- utils/utils.py:298-358  (make_grid + handel_preds)
nms()     <- utils/utils.py:67-74,232-296 (xywh2xyxy + non_max_suppression) and the greedy
             kernel of torchvision.ops.nms (third-party, NOT in /root/reference: torchvision
             pinned 0.10.0 by requirements.txt:5, 0.26.0 installed; algorithm restated in
             greedy_nms_numpy()/oracle/nms_ref.c and pinned against the installed wheel by
             tests/test_oracle_golden.py).

Deliberate omission: the reference aborts its per-image loop after 1.0 s of wall clock
(utils/utils.py:245,292-294) leaving later images empty.  That is a nondeterministic
hazard, not an algorithm; it is not restated.
"""
import ctypes
import os

import numpy as np
import torch
import torch.nn.functional as F

MAX_WH = 4096       # utils/utils.py:241
MAX_DET = 300       # utils/utils.py:242
MAX_NMS = 30000     # utils/utils.py:243


def decode(preds, cfg):
    """handel_preds (utils/utils.py:303-358) without the per-image Python loop.

    preds: 6-tuple (reg_2,obj_2,cls_2,reg_3,obj_3,cls_3) NCHW fp32 CPU tensors.
    Returns [N, sum(h*w*A), 5+C] fp32; row index within a level is (y*w + x)*A + a.
    Arithmetic follows the reference dtype flow exactly: xy in fp32; wh = fp32 (s*2)^2
    promoted to fp64 by the float64 anchors, multiplied, then rounded to fp32 on store
    (utils/utils.py:305-306,337); obj sigmoid fp32; cls softmax fp32 over classes.
    """
    A = cfg["anchor_num"]
    levels = len(preds) // 3
    anchors = torch.from_numpy(np.array(cfg["anchors"], dtype=np.float64).reshape(levels, A, 2))
    outs = []
    for i in range(levels):
        reg, obj, cls = preds[3 * i], preds[3 * i + 1], preds[3 * i + 2]
        N, _, h, w = reg.shape
        C = cls.shape[1]
        r = reg.permute(0, 2, 3, 1).reshape(N, h, w, A, 4)
        o = obj.permute(0, 2, 3, 1).reshape(N, h, w, A)
        c = cls.permute(0, 2, 3, 1)                                    # [N,h,w,C]
        gy, gx = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
        grid = torch.stack((gx, gy), 2).reshape(1, h, w, 1, 2)         # (x, y) int64
        stride = cfg["height"] / h                                     # python float, both axes
        box = torch.zeros(N, h, w, A, 5 + C, dtype=torch.float32)
        box[..., 0:2] = ((r[..., 0:2].sigmoid() * 2.0 - 0.5) + grid) * stride
        box[..., 2:4] = (r[..., 2:4].sigmoid() * 2) ** 2 * anchors[i]  # fp64 -> fp32 on store
        box[..., 4] = o.sigmoid()
        box[..., 5:] = F.softmax(c, dim=3).unsqueeze(3)                # same cls for every anchor
        outs.append(box.reshape(N, h * w * A, 5 + C))
    return torch.cat(outs, 1)


def greedy_nms_numpy(boxes, scores, iou_thres):
    """torchvision.ops.nms CPU semantics: stable descending sort, fp32 IoU
    inter/(a_i+a_j-inter) with no +1, suppress iff (double)iou > iou_thres."""
    boxes = np.ascontiguousarray(boxes, dtype=np.float32)
    scores = np.asarray(scores, dtype=np.float32)
    n = boxes.shape[0]
    order = np.argsort(-scores, kind="stable")
    x1, y1, x2, y2 = boxes[:, 0], boxes[:, 1], boxes[:, 2], boxes[:, 3]
    areas = (x2 - x1) * (y2 - y1)
    dead = np.zeros(n, dtype=bool)
    keep = []
    thr = float(iou_thres)
    for _i in range(n):
        i = order[_i]
        if dead[i]:
            continue
        keep.append(i)
        rest = order[_i + 1:]
        w = np.maximum(np.float32(0), np.minimum(x2[i], x2[rest]) - np.maximum(x1[i], x1[rest]))
        h = np.maximum(np.float32(0), np.minimum(y2[i], y2[rest]) - np.maximum(y1[i], y1[rest]))
        inter = w * h
        with np.errstate(divide="ignore", invalid="ignore"):
            ovr = inter / (areas[i] + areas[rest] - inter)
        dead[rest[ovr.astype(np.float64) > thr]] = True
    return np.asarray(keep, dtype=np.int64)


_clib = None


def _load_c():
    global _clib
    if _clib is None:
        here = os.path.dirname(os.path.abspath(__file__))
        path = os.path.join(here, "_build", "liboracle.so")
        if not os.path.exists(path):
            raise RuntimeError("oracle C library not built: run `make -C oracle` (or __graft_entry__.build())")
        lib = ctypes.CDLL(path)
        lib.oracle_nms_image.restype = ctypes.c_int
        lib.oracle_nms_image.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_float,
                                         ctypes.c_double, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                         ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p]
        _clib = lib
    return _clib


def nms_image_c(x, conf_thres, iou_thres, classes=None, max_det=MAX_DET, max_wh=MAX_WH):
    """One image through oracle/nms_ref.c.  x: [M,5+C] fp32 numpy.  Returns (rows[n,6], idx[n])."""
    lib = _load_c()
    x = np.ascontiguousarray(x, dtype=np.float32)
    M, D = x.shape
    out = np.zeros((max_det, 6), dtype=np.float32)
    idx = np.zeros(max_det, dtype=np.int32)
    if classes is None:
        cls_arr, ncls, cls_ptr = None, 0, None
    else:
        cls_arr = np.ascontiguousarray(classes, dtype=np.int32)
        ncls, cls_ptr = cls_arr.size, cls_arr.ctypes.data
    n = lib.oracle_nms_image(x.ctypes.data, M, D - 5, conf_thres, iou_thres, cls_ptr, ncls, max_det, max_wh,
                             out.ctypes.data, idx.ctypes.data)
    if n < 0:
        raise RuntimeError("oracle_nms_image failed (%d)" % n)
    return out[:n].copy(), idx[:n].copy()


def nms(prediction, conf_thres=0.3, iou_thres=0.45, classes=None, return_indices=False, impl="c", max_det=MAX_DET,
        max_wh=MAX_WH):
    """non_max_suppression (utils/utils.py:232-296): list of [n_i,6] fp32 CPU tensors
    (x1,y1,x2,y2,conf,cls) sorted by descending conf, at most max_det (the reference: 300) per image.
    max_wh is the per-class box offset of utils/utils.py:283 (the reference: 4096).

    impl="c" uses oracle/nms_ref.c, impl="numpy" the numpy restatement (slow, tests only).
    With return_indices also returns, per image, the row indices into prediction[i]."""
    pred = prediction.detach().cpu().numpy() if isinstance(prediction, torch.Tensor) else np.asarray(prediction)
    outs, idxs = [], []
    for x in pred:
        if impl == "c":
            rows, idx = nms_image_c(x, conf_thres, iou_thres, classes, max_det, max_wh)
        else:
            rows, idx = _nms_image_numpy(x, conf_thres, iou_thres, classes, max_det, max_wh)
        outs.append(torch.from_numpy(rows).reshape(-1, 6))
        idxs.append(idx.astype(np.int64))
    return (outs, idxs) if return_indices else outs


def _nms_image_numpy(x, conf_thres, iou_thres, classes=None, max_det=MAX_DET, max_wh=MAX_WH):
    x = np.asarray(x, dtype=np.float32)
    ct = np.float32(conf_thres)                            # torch compares the fp32 tensor with float32(thres)
    src = np.nonzero(x[:, 4] > ct)[0]                      # utils/utils.py:254
    x = x[src]
    if x.shape[0] == 0:
        return np.zeros((0, 6), np.float32), np.zeros(0, np.int64)
    prob = x[:, 5:] * x[:, 4:5]                            # :261 conf = obj*cls, fp32
    half_w, half_h = x[:, 2] / np.float32(2), x[:, 3] / np.float32(2)
    box = np.stack((x[:, 0] - half_w, x[:, 1] - half_h, x[:, 0] + half_w, x[:, 1] + half_h), 1)  # :67-74
    j = prob.argmax(1)                                     # first max, :267
    conf = prob[np.arange(prob.shape[0]), j]
    m = conf > ct                              # :268
    if classes is not None:
        m &= np.isin(j, np.asarray(classes))               # :271-272
    box, conf, j, src = box[m], conf[m], j[m], src[m]
    if box.shape[0] == 0:
        return np.zeros((0, 6), np.float32), np.zeros(0, np.int64)
    if box.shape[0] > MAX_NMS:                             # :278-280
        top = np.argsort(-conf, kind="stable")[:MAX_NMS]
        box, conf, j, src = box[top], conf[top], j[top], src[top]
    off = (j.astype(np.float32) * np.float32(max_wh))[:, None]                # :283
    keep = greedy_nms_numpy(box + off, conf, iou_thres)[:max_det]             # :285-288
    rows = np.concatenate((box[keep], conf[keep, None], j[keep, None].astype(np.float32)), 1)
    return rows.astype(np.float32), src[keep]

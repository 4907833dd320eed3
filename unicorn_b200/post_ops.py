"""Wrappers of the detector's post-processing entry points (include/unicorn_b200.h: uc_postprocess_batched_ex,
uc_det_candidates_batched, uc_postprocess_nms_batched), next to the ones of unicorn_b200.ops that the tracking frames use.  Their
results are pinned bit for bit to head_decode + postprocess_device (tests/test_det_gpu.py)."""
import ctypes

import torch

from . import _lib
from .ops import _L, _S, _f, _l, _p

POST_CLASS_AGNOSTIC = 1  # UC_POST_CLASS_AGNOSTIC


def postprocess_device_ex(pred, ncls, conf, nms, ws, max_keep=0, class_agnostic=False):
    """postprocess_device with the NMS mode: class_agnostic=True suppresses across classes (postprocess(..., class_agnostic=True)).
    pred fp32 [B, A, 5+ncls] (or [A, 5+ncls] with a workspace of batch 1)."""
    assert pred.is_contiguous() and pred.dtype == torch.float32 and pred.shape[-2] == ws.max_anchors
    B = pred.shape[0] if pred.dim() == 3 else 1
    assert B == ws.batch, "postprocess_device_ex: a batch of B images needs a PostWorkspace(A, device, batch=B)"
    _lib.check(_L().uc_postprocess_batched_ex(_p(pred), ws.max_anchors, ncls, _f(conf), _f(nms), int(max_keep), B,
                                              POST_CLASS_AGNOSTIC if class_agnostic else 0, _p(ws.buf), _l(ws.nbytes), _p(ws.dets),
                                              _p(ws.count), _p(ws.anchors), _S()), "uc_postprocess_batched_ex", 4)
    return ws.dets, ws.count


def det_candidates(regobj, cls, hw, strides, ncls, conf, ws):
    """Decode + score filter of B images straight from the head maps (NHWC fp32 [B,h,w,ld] per level, as head_decode takes them)
    into the workspace, without the decoded tensor: what head_decode + the filter of postprocess_device leave there.  Follow with
    postprocess_nms."""
    B = regobj[0].shape[0]
    A = sum(h * w for h, w in hw)
    assert all(t.dim() == 4 and t.shape[0] == B and t.dtype == torch.float32 for t in list(regobj) + list(cls))
    assert B == ws.batch and A == ws.max_anchors, "det_candidates: a batch of B images needs a PostWorkspace(A, device, batch=B)"
    ro = (ctypes.c_void_p * 3)(*[t.data_ptr() for t in regobj])
    cl = (ctypes.c_void_p * 3)(*[t.data_ptr() for t in cls])
    hwa = (ctypes.c_int * 6)(*[v for pair in hw for v in pair])
    st = (ctypes.c_int * 3)(*strides)
    bs_ro = (ctypes.c_long * 3)(*[t.stride(0) for t in regobj])
    bs_cl = (ctypes.c_long * 3)(*[t.stride(0) for t in cls])
    _lib.check(_L().uc_det_candidates_batched(ro, cl, hwa, st, regobj[0].shape[-1], cls[0].shape[-1], bs_ro, bs_cl, ncls, B, _f(conf),
                                              _p(ws.buf), _l(ws.nbytes), _S()), "uc_det_candidates_batched")


def postprocess_nms(nms, ws, max_keep=0, class_agnostic=False):
    """Sort, gather and greedy NMS of the candidates det_candidates left in ws; ws.dets / ws.count hold the result."""
    _lib.check(_L().uc_postprocess_nms_batched(ws.max_anchors, _f(nms), int(max_keep), ws.batch, POST_CLASS_AGNOSTIC if class_agnostic else 0,
                                               _p(ws.buf), _l(ws.nbytes), _p(ws.dets), _p(ws.count), _p(ws.anchors), _S()),
               "uc_postprocess_nms_batched")
    return ws.dets, ws.count

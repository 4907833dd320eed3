"""Wrappers of the detector's post-processing entry points (include/unicorn_b200.h: uc_postprocess_batched_ex,
uc_det_candidates_batched, uc_postprocess_nms_batched, and for the instance segmenter uc_dynamic_masks_batched over a window of NMS
rows and uc_inst_encode_batched; for the BDD100K MOTS bitmasks uc_bdd_bitmask_batched), next to the ones of unicorn_b200.ops that the
tracking frames use.  The detector's results are pinned bit for bit to head_decode + postprocess_device (tests/test_det_gpu.py)."""
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


def dynamic_masks_rows(mask_feats, up_masks, dyn_levels, level_hw, anchors, count, image_of, n_max, up_rate, out, scratch,
                       soi=(64.0, 128.0, 256.0)):
    """uc_dynamic_masks_batched with d_rate = 1 for a window of NMS rows: image b's masks of rows row0 .. row0 + count[b] - 1, where
    `anchors` is the [B, A] NMS anchor buffer viewed from column row0 (its image stride stays A) and count device int32 [B] holds
    each image's rows in the window (at most n_max); image_of: device int32 [0, 1, ..., B-1].  mask_feats fp32 [B,h,w,8], up_masks fp32 [B,h,w,9*up^2]; out fp32
    [B, n_max, h*up, w*up]; scratch >= B*n_max*h*w floats (the logits; d_rate = 1 needs no upsampling buffer)."""
    B, h, w, _ = mask_feats.shape
    assert mask_feats.is_contiguous() and up_masks.is_contiguous() and up_masks.shape[:3] == (B, h, w)
    assert all(t.shape[0] == B and t.stride(-1) == 1 for t in dyn_levels) and anchors.dim() == 2 and anchors.shape[0] == B
    assert count.dtype == torch.int32 and count.numel() == B and scratch.numel() >= B * n_max * h * w
    assert out.shape == (B, n_max, h * up_rate, w * up_rate) and out.is_contiguous() and out.dtype == torch.float32
    dl = (ctypes.c_void_p * 3)(*[t.data_ptr() for t in dyn_levels])
    hw = (ctypes.c_int * 6)(*[v for pair in level_hw for v in pair])
    bs = (ctypes.c_long * 3)(*[t.stride(0) for t in dyn_levels])
    assert image_of.dtype == torch.int32 and image_of.numel() == B
    _lib.check(_L().uc_dynamic_masks_batched(_p(mask_feats), _p(up_masks), B, h, w, up_rate, 1, dl, dyn_levels[0].shape[-1], bs, hw,
                                             (ctypes.c_int * 3)(8, 16, 32), (ctypes.c_float * 3)(*soi), _p(anchors), _l(anchors.stride(0)),
                                             _p(count), _p(image_of), B, n_max, _p(scratch), _p(out), _S()), "uc_dynamic_masks_batched", 2)
    return out


def inst_encode(maps, count, row0, d_rate, thr, r, H, W, ws, emit, chars, offsets):
    """COCO RLE strings of the masks of NMS rows row0 .. row0 + n_max - 1 of B images (uc_inst_encode_batched): maps fp32
    [B, n_max, hs, ws], the d_rate = 1 output of dynamic_masks_rows, upsampled x d_rate, resized by 1/r[b] to the original H[b] x W[b],
    thresholded at thr and encoded over the whole frame.  count: device int32 [B], every image's NMS row count.  r, H, W: B host
    values.  emit uint8 [>= B*n_max], offsets int64 [>= B*n_max + 1] device outputs; chars: uint8 device buffer (its size is the
    capacity), nothing past it is written.  Launches only: offsets[B*n_max] is the number of chars needed."""
    B, n_max, hs, wsz = maps.shape
    assert maps.dtype == torch.float32 and maps.stride(3) == 1 and maps.stride(2) == wsz and maps.stride(1) == hs * wsz
    assert count.dtype == torch.int32 and count.numel() >= B and len(r) == len(H) == len(W) == B
    assert emit.dtype == torch.uint8 and emit.numel() >= B * n_max and offsets.dtype == torch.int64 and offsets.numel() >= B * n_max + 1
    assert chars.dtype == torch.uint8 and ws.dtype == torch.uint8
    ints = lambda v: (ctypes.c_int * B)(*[int(x) for x in v])  # noqa: E731
    _lib.check(_L().uc_inst_encode_batched(_p(maps), _l(maps.stride(0)), n_max, hs, wsz, int(d_rate), B, _p(count), int(row0), ints(H), ints(W),
                                           (ctypes.c_double * B)(*[float(x) for x in r]), _f(thr), _p(ws), _l(ws.numel()), _p(emit),
                                           _p(chars), _l(chars.numel()), _p(offsets), _S()), "uc_inst_encode_batched", 3)
    return offsets


BDD_BAD_CHARS, BDD_BAD_RUNS, BDD_BAD_INDEX = 1, 2, 4  # UC_BDD_* status flags


def _ints(v, ctype=ctypes.c_int):
    return (ctype * len(v))(*[int(x) for x in v])


def bdd_bitmask_workspace_bytes(k, H, W, n_chars):
    """uc_bdd_bitmask_workspace_bytes: the workspace of a uc_bdd_bitmask_batched call on frames with k[b] instances of H[b] x W[b]
    and n_chars chars in all."""
    n = _L().uc_bdd_bitmask_workspace_bytes
    n.restype = ctypes.c_long
    nbytes = n(len(k), _ints(k), _ints(H), _ints(W), _l(n_chars))
    if nbytes < 0:
        raise ValueError(f"bdd_bitmask_workspace_bytes: bad arguments k={list(k)}, H={list(H)}, W={list(W)}, n_chars={n_chars}")
    return nbytes


def bdd_bitmask(chars, n_chars, offsets, colors, ranks, k, H, W, out, out_offsets, ws, status):
    """The RGBA bitmasks of B frames (uc_bdd_bitmask_batched): chars uint8 (the first n_chars used), offsets int64 [K+1], colors int32
    [K] (packed R | G << 8 | B << 16 | A << 24) and ranks int32 [K] on the device, K = sum(k); k, H, W: B host ints.  Frame b is
    written as uint8 [H[b], W[b], 4] at byte out_offsets[b] (host) of the device buffer out.  status: device int32 [>= B], frame b's
    UC_BDD_* flags (0 = every string well formed).  ws: device uint8, bdd_bitmask_workspace_bytes(k, H, W, n_chars) bytes.  Launches
    only."""
    B = len(k)
    assert len(H) == len(W) == len(out_offsets) == B and sum(k) + 1 <= offsets.numel()
    assert chars.dtype == torch.uint8 and n_chars <= chars.numel() and offsets.dtype == torch.int64
    assert colors.dtype == ranks.dtype == status.dtype == torch.int32 and colors.numel() >= sum(k) and ranks.numel() >= sum(k)
    assert out.dtype == ws.dtype == torch.uint8 and status.numel() >= B
    _lib.check(_L().uc_bdd_bitmask_batched(B, _ints(k), _ints(H), _ints(W), _ints(out_offsets, ctypes.c_long), _p(chars), _l(n_chars),
                                           _p(offsets), _p(colors), _p(ranks), _p(ws), _l(ws.numel()), _p(out), _l(out.numel()), _p(status),
                                           _S()), "uc_bdd_bitmask_batched", 3 if sum(k) else 1)
    return status

"""Wrappers of uc_groupnorm_apply_gather, the stem of UnicornEngine.head_shared, of uc_vos_aggregate_batched, the result
assembly of UnicornUnifiedMaskBatch, and of uc_letterbox_nv12, the letterbox of NV12 frames (include/unicorn_b200.h).  They sit next
to unicorn_b200.ops rather than in it because every launcher of ops has a per-launch fp32 reference in the tracking-frame launch check
(tests/test_launch_parity_gpu.py); these are pinned bit for bit instead: to their B = 1 launches, ops.groupnorm_apply
(tests/test_unified_gpu.py, tests/test_unified_batch_gpu.py) and ops.vos_aggregate (tests/test_unified_mask_batch_gpu.py), and to
cv2's conversion followed by the reference's letterbox (tests/test_nv12_gpu.py)."""
import ctypes

import torch

from . import _lib
from .ops import _L, _S, _f, _l, _nhwc_ld, _p, _vos_objects


def groupnorm_apply_gather(x, stats, w, b, G, eps, act, out, n_plain, src_of, prior=None, beta=None):
    """x NHWC view of n_src images, stats their [n_src, G, 2] statistics -> out [B,H,W,C]: image b normalises image src_of[b] (a
    device int32 [B] table, read when the kernel runs; an entry outside [0, n_src) leaves image b untouched), images b < n_plain
    without a prior, images b >= n_plain with prior plane b - n_plain.  Each image equals groupnorm_apply of x[src_of[b]] at B = 1."""
    n_src, H, W, C = x.shape
    B = out.shape[0]
    assert out.shape[1:] == x.shape[1:] and out.dtype == x.dtype == torch.bfloat16
    assert stats.dtype == torch.int64 and stats.is_contiguous() and stats.numel() == n_src * G * 2
    assert src_of.dtype == torch.int32 and src_of.is_cuda and src_of.is_contiguous() and src_of.numel() == B
    if prior is not None:
        assert prior.dtype == torch.float32 and prior.is_contiguous() and prior.numel() == (B - n_plain) * H * W
    _lib.check(_L().uc_groupnorm_apply_gather(_p(x), _nhwc_ld(x), n_src, _p(stats), _p(w), _p(b), _p(out), _nhwc_ld(out), B, int(n_plain),
                                              _p(src_of), _l(H * W), C, G, _f(eps), act, _p(prior), _p(beta), _S()),
               "uc_groupnorm_apply_gather")
    return out


def vos_aggregate_batched(videos, Hin, Win):
    """vos_aggregate of several videos in one launch (uc_vos_aggregate_batched): videos is a list of (masks, init_mask, ids, r, soft,
    seg), one entry per video in the shape vos_aggregate takes (soft may be None).  Each video's seg and soft equal its own
    vos_aggregate call, bit for bit."""
    B = len(videos)
    descs = (_lib.UcVosVideo * B)()
    keep = []  # the object arrays stay alive until the call has read them
    for b, (masks, init_mask, ids, r, soft, seg) in enumerate(videos):
        objs, n, H0, W0 = _vos_objects(masks, init_mask, ids, Hin, Win, soft, seg)
        keep.append(objs)
        descs[b].objs = ctypes.cast(objs, ctypes.POINTER(_lib.UcVosObject))
        descs[b].n, descs[b].H, descs[b].W, descs[b].r = n, H0, W0, float(r)
        descs[b].soft_out, descs[b].seg_out = _p(soft), _p(seg)
    _lib.check(_L().uc_vos_aggregate_batched(descs, B, Hin, Win, _S()), "uc_vos_aggregate_batched")
    return [v[5] for v in videos]


def letterbox_nv12(src, input_size, pad=114, out=None):
    """src: NV12 uint8 [3h/2, w] CUDA tensor (h rows of Y, then h/2 rows of interleaved U, V; unit column stride, any row stride
    >= w, so a view of a wider decoder surface works) -> (uint8 [1,H,W,3] letterboxed frame, r): ops.letterbox_u8's output, with r and
    the resized size computed as it computes them, for the BGR frame cv2.cvtColor(COLOR_YUV2BGR_NV12) makes of src."""
    if not torch.is_tensor(src) or src.dtype != torch.uint8 or src.dim() != 2 or src.shape[0] < 3 or src.shape[0] % 3 or src.shape[1] < 1:
        raise ValueError(f"letterbox_nv12: src must be an NV12 uint8 [3h/2, w] tensor, got {getattr(src, 'shape', type(src))} "
                         f"{getattr(src, 'dtype', '')}")
    if src.stride(1) != 1 or src.stride(0) < src.shape[1] or not src.is_cuda:
        raise ValueError(f"letterbox_nv12: src must be a CUDA tensor with unit column stride and a row stride >= w, got {src.device}, "
                         f"strides {src.stride()}")
    h, w = src.shape[0] * 2 // 3, src.shape[1]
    H, W = input_size
    r = min(H / h, W / w)
    if out is None:
        out = torch.empty(1, H, W, 3, dtype=torch.uint8, device=src.device)
    if out.dtype != torch.uint8 or tuple(out.shape) != (1, H, W, 3) or not out.is_contiguous() or out.device != src.device:
        raise ValueError(f"letterbox_nv12: out must be a contiguous uint8 [1, {H}, {W}, 3] tensor on {src.device}, got "
                         f"{tuple(out.shape)} {out.dtype} on {out.device}")
    ld = src.stride(0)
    _lib.check(_L().uc_letterbox_nv12(_p(src), ctypes.c_void_p(src.data_ptr() + h * ld), ld, h, w, _p(out), H, W, int(h * r), int(w * r),
                                      int(pad), _S()), "uc_letterbox_nv12")
    return out, r

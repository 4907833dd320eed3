"""Wrappers of uc_groupnorm_apply_gather, the stem of UnicornEngine.head_shared, and of uc_vos_aggregate_batched, the result
assembly of UnicornUnifiedMaskBatch (include/unicorn_b200.h).  They sit next to unicorn_b200.ops rather than in it because every
launcher of ops has a per-launch fp32 reference in the tracking-frame launch check (tests/test_launch_parity_gpu.py); these are
pinned bit for bit to their B = 1 launches instead: ops.groupnorm_apply (tests/test_unified_gpu.py, tests/test_unified_batch_gpu.py)
and ops.vos_aggregate (tests/test_unified_mask_batch_gpu.py)."""
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

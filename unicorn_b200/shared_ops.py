"""Wrapper of uc_groupnorm_apply_bcast, the stem of UnicornEngine.head_shared (include/unicorn_b200.h).  It sits next to
unicorn_b200.ops rather than in it because every launcher of ops has a per-launch fp32 reference in the tracking-frame launch check
(tests/test_launch_parity_gpu.py); this one is pinned bit for bit to ops.groupnorm_apply at B = 1 instead (tests/test_unified_gpu.py)."""
import torch

from . import _lib
from .ops import _L, _S, _f, _l, _nhwc_ld, _p


def groupnorm_apply_bcast(x, stats, w, b, G, eps, act, out, n_plain, prior=None, beta=None):
    """x NHWC view of ONE image, stats its [G, 2] statistics -> out [B,H,W,C]: images b < n_plain without a prior, images b >= n_plain
    with prior plane b - n_plain (prior fp32, (B - n_plain) * H * W elements).  Each image equals groupnorm_apply of x at B = 1."""
    _, H, W, C = x.shape
    B = out.shape[0]
    assert x.shape[0] == 1 and out.shape[1:] == x.shape[1:] and out.dtype == x.dtype == torch.bfloat16
    if prior is not None:
        assert prior.dtype == torch.float32 and prior.is_contiguous() and prior.numel() == (B - n_plain) * H * W
    _lib.check(_L().uc_groupnorm_apply_bcast(_p(x), _nhwc_ld(x), _p(stats), _p(w), _p(b), _p(out), _nhwc_ld(out), B, int(n_plain),
                                             _l(H * W), C, G, _f(eps), act, _p(prior), _p(beta), _S()), "uc_groupnorm_apply_bcast")
    return out

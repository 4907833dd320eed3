"""Python wrappers over the C ABI.  Tensors are torch CUDA tensors used purely as device memory:
activations are NHWC views (B, H, W, C) with unit channel stride and a constant pixel stride (so a channel
slice of a wider buffer is a valid operand, which is how concatenations are formed without copies)."""
import ctypes

import torch

from . import _lib
from ._lib import BF16, F32, F16, ACT_NONE, ACT_RELU, ACT_GELU, ACT_SILU, ACT_SIGMOID  # noqa: F401

_DT = {torch.bfloat16: BF16, torch.float32: F32, torch.float16: F16}


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _nhwc_ld(t):
    """pixel stride of an NHWC view; validates the layout."""
    assert t.dim() == 4 and t.is_cuda, "expected a CUDA NHWC tensor"
    B, H, W, C = t.shape
    ld = t.stride(2) if W > 1 else (t.stride(1) // W if H > 1 else max(C, t.stride(2)))
    assert t.stride(3) == 1 or C == 1
    if W > 1:
        assert t.stride(2) == ld
    if H > 1:
        assert t.stride(1) == W * ld, (t.shape, t.stride())
    if B > 1:
        assert t.stride(0) == H * W * ld
    return ld


def pack_conv_weight(w, dtype=torch.bfloat16, cout_pad=8):
    """[Cout, Cin, KH, KW] (or [Cout, Cin] for Linear) fp32 -> [Cout_pad, KH*KW, Cin] 16-bit, K-major."""
    if w.dim() == 2:
        w = w[:, :, None, None]
    Cout, Cin, KH, KW = w.shape
    Cp = (Cout + cout_pad - 1) // cout_pad * cout_pad
    out = torch.zeros(Cp, KH * KW, Cin, dtype=dtype, device=w.device)
    out[:Cout] = w.permute(0, 2, 3, 1).reshape(Cout, KH * KW, Cin).to(dtype)
    return out.contiguous()


CONV_TRACE = None


def conv2d(x, w_packed, KH, KW, stride=1, pad=0, bias=None, act=ACT_NONE, gamma=None, res=None, out=None,
           out_dtype=None, block_n=0, gn_stats=None, gn_groups=0, row_stats=None, col_s=None, row_eps=1e-6, act_after_res=False):
    """x: NHWC view (B,H,W,Cin) bf16/f16.  w_packed: [Cout, KH*KW, Cin].  Returns NHWC (B,Ho,Wo,Cout).
    act_after_res=True (with act=ACT_RELU and res): y = relu(conv + bias + res) instead of res + act(conv + bias)."""
    B, H, W, Cin = x.shape
    Cout = w_packed.shape[0]
    assert w_packed.shape[1] == KH * KW and w_packed.shape[2] == Cin and w_packed.is_contiguous()
    assert w_packed.dtype == x.dtype
    Ho = (H + 2 * pad - KH) // stride + 1
    Wo = (W + 2 * pad - KW) // stride + 1
    if out is None:
        out = torch.empty(B, Ho, Wo, Cout, dtype=out_dtype or x.dtype, device=x.device)
    assert out.shape == (B, Ho, Wo, Cout), (out.shape, (B, Ho, Wo, Cout))
    d = _lib.UcConv2d()
    d.x, d.x_dtype = _p(x), _DT[x.dtype]
    d.B, d.H, d.W, d.Cin, d.ldx = B, H, W, Cin, _nhwc_ld(x)
    d.w = _p(w_packed)
    d.Cout, d.KH, d.KW, d.stride, d.pad = Cout, KH, KW, stride, pad
    d.bias, d.act, d.gamma = _p(bias), act, _p(gamma)
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.numel() >= Cout
    if gamma is not None:
        assert gamma.dtype == torch.float32 and gamma.numel() >= Cout
    d.res, d.ldres = _p(res), (_nhwc_ld(res) if res is not None else 0)
    if res is not None:
        assert res.dtype == out.dtype and res.shape == out.shape
    d.y, d.ldy, d.y_dtype = _p(out), _nhwc_ld(out), _DT[out.dtype]
    d.block_n = block_n
    d.gn_stats, d.gn_groups = _p(gn_stats), gn_groups
    d.row_stats, d.col_s, d.row_eps = _p(row_stats), _p(col_s), row_eps
    d.act_after_res = int(bool(act_after_res))
    if row_stats is not None:
        assert row_stats.dtype == torch.int64 and row_stats.numel() == B * H * W * 2 and col_s is not None and col_s.numel() >= Cout
    if CONV_TRACE is not None:  # tools/profile_frame.py: conv launches in issue order, to label an ncu launch list
        CONV_TRACE.append(dict(M=B * Ho * Wo, N=Cout, K=Cin * KH * KW, k=KH, s=stride, bn=block_n, act=act, gn=gn_groups,
                               f32=int(out.dtype == torch.float32)))
    _lib.check(_lib.lib().uc_conv2d(ctypes.byref(d), _lib.stream_ptr()), "uc_conv2d")
    return out


def linear(x2d, w_packed, **kw):
    """x2d: [M, K] rows (unit inner stride).  Returns [M, N]."""
    M, K = x2d.shape
    assert x2d.stride(1) == 1
    x4 = x2d.as_strided((1, 1, M, K), (M * x2d.stride(0), M * x2d.stride(0), x2d.stride(0), 1))
    out = kw.pop("out", None)
    res = kw.pop("res", None)
    if out is not None:
        out = out.as_strided((1, 1, M, out.shape[1]), (M * out.stride(0), M * out.stride(0), out.stride(0), 1))
    if res is not None:
        res = res.as_strided((1, 1, M, res.shape[1]), (M * res.stride(0), M * res.stride(0), res.stride(0), 1))
    y = conv2d(x4, w_packed, 1, 1, out=out, res=res, **kw)
    return y.as_strided((M, y.shape[3]), (y.stride(2), 1))


# ------------------------------------------------------------------------------------------- other entry points
def _L():
    return _lib.lib()


def _S():
    return _lib.stream_ptr()


_f = ctypes.c_float
_i = ctypes.c_int
_l = ctypes.c_long


def pack_stem_weight(w):
    """[C0,3,4,4] -> [48, C0] fp32 (k = (ci*4+kh)*4+kw)."""
    return w.reshape(w.shape[0], 48).t().contiguous().float()


def pack_dw_weight(w):
    """[C,1,7,7] -> [49, C] fp32."""
    return w.reshape(w.shape[0], 49).t().contiguous().float()


def pack_dw_weight_mma(w, bias):
    """[C,1,7,7], [C] -> int32 [ceil(C/32), 1824]: per 32-channel chunk the bf16 tap pairs {e[j-1], e[j]}, j = 0..7, of every channel
    and filter row ([32][7][8] words; e = the row padded with zeros, lower index in the low half) followed by the 32 fp32 biases; zero
    for the channels that pad C to a multiple of 32 — the operand of uc_dwconv7_mma, which builds the B fragments of its Toeplitz
    blocks T[k][n] = e[k-n-1] from it."""
    C = w.shape[0]
    Cp = -(-C // 32) * 32
    e = torch.zeros(Cp, 7, 9, dtype=torch.bfloat16, device=w.device)  # e[-1] .. e[7]
    e[:C, :, 1:8] = w.reshape(C, 7, 7).to(torch.bfloat16)
    bits = e.view(torch.int16).to(torch.int32) & 0xffff
    pairs = (bits[:, :, 0:8] | (bits[:, :, 1:9] << 16)).to(torch.int32).reshape(Cp // 32, 32 * 7 * 8)
    bp = torch.zeros(Cp, dtype=torch.float32, device=w.device)
    bp[:C] = bias.float()
    return torch.cat([pairs, bp.view(torch.int32).reshape(Cp // 32, 32)], dim=1).contiguous()


def dwconv7_mma(x, qtab, out=None, work_counter=None):
    B, H, W, C = x.shape
    assert x.is_contiguous() and x.dtype == torch.bfloat16 and qtab.dtype == torch.int32 and qtab.shape == (-(-C // 32), 1824)
    if out is None:
        out = torch.empty_like(x)
    _lib.check(_L().uc_dwconv7_mma(_p(x), _p(qtab), _p(out), B, H, W, C, _p(work_counter), _S()), "uc_dwconv7_mma")
    return out


def convnext_mlp_supported(C):
    return bool(_L().uc_convnext_mlp_supported(int(C)))


def convnext_mlp(t, w1f, c1, w2, b2, gamma, x, eps=1e-6):
    """x[M,C] += gamma * (W2 . GELU(W1f . LN0(t) + c1) + b2) in one launch (uc_convnext_mlp); t, x: [M, C] bf16 contiguous."""
    M, C = t.shape
    assert t.is_contiguous() and x.is_contiguous() and x.shape == t.shape and t.dtype == x.dtype == torch.bfloat16
    assert w1f.dtype == torch.bfloat16 and w1f.numel() == 4 * C * C and w2.dtype == torch.bfloat16 and w2.numel() == 4 * C * C
    _lib.check(_L().uc_convnext_mlp(_p(t), _p(w1f), _p(c1), _p(w2), _p(b2), _p(gamma), _p(x), M, C, ctypes.c_float(eps), _S()), "uc_convnext_mlp")
    return x


def stem_ln(img, w48, bias, lnw, lnb, eps=1e-6):
    """img: fp32 NCHW [B,3,H,W] or uint8 NHWC [B,H,W,3] (BGR)."""
    u8 = img.dtype == torch.uint8
    if u8:
        B, H, W, _ = img.shape
    else:
        B, _, H, W = img.shape
        assert img.dtype == torch.float32
    assert img.is_contiguous()
    C0 = w48.shape[1]
    out = torch.empty(B, H // 4, W // 4, C0, dtype=torch.bfloat16, device=img.device)
    _lib.check(_L().uc_stem_ln(_p(img), int(u8), _p(w48), _p(bias), _p(lnw), _p(lnb), _p(out), B, H, W, C0, _f(eps), _S()), "uc_stem_ln")
    return out


def pack_resnet_stem_weight(w):
    """[64,3,7,7] fp32 (BatchNorm already folded in) -> [64, 160] fp16, k = ci*49 + kh*7 + kw, zero for k >= 147."""
    out = torch.zeros(w.shape[0], 160, dtype=torch.float16, device=w.device)
    out[:, :147] = w.reshape(w.shape[0], 147).to(torch.float16)
    return out


def resnet_stem(img, w160, bias, out=None):
    """conv7x7s2 + bias + ReLU + maxpool3x3s2 in one launch.  img: fp32 NCHW [B,3,H,W] or uint8 NHWC [B,H,W,3] (BGR).
    Returns NHWC bf16 [B,H/4,W/4,64]."""
    u8 = img.dtype == torch.uint8
    if u8:
        B, H, W, _ = img.shape
    else:
        B, _, H, W = img.shape
        assert img.dtype == torch.float32
    assert img.is_contiguous() and w160.dtype == torch.float16 and w160.shape == (64, 160) and bias.dtype == torch.float32
    if out is None:
        out = torch.empty(B, H // 4, W // 4, 64, dtype=torch.bfloat16, device=img.device)
    assert out.shape == (B, H // 4, W // 4, 64) and out.is_contiguous() and out.dtype == torch.bfloat16
    _lib.check(_L().uc_resnet_stem(_p(img), int(u8), _p(w160), _p(bias), _p(out), B, H, W, _S()), "uc_resnet_stem")
    return out


def dwconv7_ln(x, w49, bias, lnw, lnb, eps=1e-6, out=None):
    B, H, W, C = x.shape
    assert x.is_contiguous() and x.dtype == torch.bfloat16
    if out is None:
        out = torch.empty_like(x)
    _lib.check(_L().uc_dwconv7_ln(_p(x), _p(w49), _p(bias), _p(lnw), _p(lnb), _p(out), B, H, W, C, _f(eps), _S()), "uc_dwconv7_ln")
    return out


def dwconv7(x, w49, bias, out=None, ln_stats=None, work_counter=None):
    B, H, W, C = x.shape
    assert x.is_contiguous() and x.dtype == torch.bfloat16
    if out is None:
        out = torch.empty_like(x)
    if ln_stats is not None:
        assert ln_stats.dtype == torch.int64 and ln_stats.is_contiguous() and ln_stats.numel() == B * H * W * 2
    if work_counter is not None:
        assert work_counter.dtype == torch.int32 and work_counter.numel() >= 1
    _lib.check(_L().uc_dwconv7(_p(x), _p(w49), _p(bias), _p(out), B, H, W, C, _p(ln_stats), _p(work_counter), _S()), "uc_dwconv7")
    return out


def layernorm(x2d, w, b, eps, res=None, out=None):
    """rows [M, C] (unit inner stride)."""
    M, C = x2d.shape
    if out is None:
        out = torch.empty(M, C, dtype=x2d.dtype, device=x2d.device)
    _lib.check(_L().uc_layernorm(_p(x2d), x2d.stride(0), _p(res), res.stride(0) if res is not None else 0, _p(w), _p(b),
                                 _p(out), out.stride(0), _l(M), C, _f(eps), _DT[x2d.dtype], _S()), "uc_layernorm")
    return out


def groupnorm_apply(x, stats, w, b, G, eps, act, out=None, prior=None, beta=None, add2=None, out2=None):
    """x NHWC view; in-place when out is None."""
    B, H, W, C = x.shape
    if out is None:
        out = x
    ld2 = _nhwc_ld(add2) if add2 is not None else 0
    _lib.check(_L().uc_groupnorm_apply(_p(x), _nhwc_ld(x), _p(stats), _p(w), _p(b), _p(out), _nhwc_ld(out), B, _l(H * W), C, G,
                                       _f(eps), act, _p(prior), _p(beta), _p(add2), ld2, _p(out2),
                                       _nhwc_ld(out2) if out2 is not None else 0, _S()), "uc_groupnorm_apply")
    return out


def copy_upsample(src, dst, up):
    B, Hs, Ws, C = src.shape
    assert dst.shape == (B, Hs * up, Ws * up, C)
    _lib.check(_L().uc_copy_upsample(_p(src), _nhwc_ld(src), _p(dst), _nhwc_ld(dst), B, Hs, Ws, C, up, _S()), "uc_copy_upsample")
    return dst


def pixel_shuffle2(x, out=None):
    B, H, W, C4 = x.shape
    Co = C4 // 4
    if out is None:
        out = torch.empty(B, 2 * H, 2 * W, Co, dtype=x.dtype, device=x.device)
    _lib.check(_L().uc_pixel_shuffle2(_p(x), _nhwc_ld(x), _p(out), _nhwc_ld(out), B, H, W, Co, _S()), "uc_pixel_shuffle2")
    return out


def bilinear(src, Hd, Wd, scale_h=0.0, scale_w=0.0, out=None):
    """src fp32 [..., Hs, Ws] contiguous planes."""
    Hs, Ws = src.shape[-2:]
    P = src.numel() // (Hs * Ws)
    if out is None:
        out = torch.empty(*src.shape[:-2], Hd, Wd, dtype=torch.float32, device=src.device)
    _lib.check(_L().uc_bilinear_f32(_p(src), _p(out), P, Hs, Ws, Hd, Wd, _f(scale_h), _f(scale_w), _S()), "uc_bilinear_f32")
    return out


def add(a2d, b2d, out=None):
    M, C = a2d.shape
    if out is None:
        out = torch.empty(M, C, dtype=a2d.dtype, device=a2d.device)
    _lib.check(_L().uc_add(_p(a2d), a2d.stride(0), _p(b2d), b2d.stride(0), _p(out), out.stride(0), _l(M), C, _DT[a2d.dtype], _S()), "uc_add")
    return out


def copy_rows_if(flag, src, dst, invert=False, gate=None):
    """dst <- src (NHWC views of equal shape, channel-contiguous) when (flag[0] != 0) != invert — decided on the device.
    With B > 1 images ([B,h,w,C] maps, flag int32 [B]) or a gate (int32 [B]), image b is copied when (gate is None or gate[b] != 0)
    and (flag[b] != 0) != invert, all images in one launch."""
    assert src.shape == dst.shape and src.dtype == dst.dtype and flag.dtype == torch.int32
    B, C = src.shape[0], src.shape[-1]
    es = src.element_size()
    if B == 1 and gate is None:
        rows = src.numel() // C
        _lib.check(_L().uc_copy_rows_if(_p(flag), int(bool(invert)), _p(src), _l(_nhwc_ld(src) * es), _p(dst), _l(_nhwc_ld(dst) * es), _l(rows), C * es, _S()),
                   "uc_copy_rows_if")
        return dst
    assert src.dim() == 4 and flag.numel() == B and (gate is None or (gate.dtype == torch.int32 and gate.numel() == B))
    rows = src.numel() // (B * C)
    lds, ldd = _nhwc_ld(src), _nhwc_ld(dst)
    _lib.check(_L().uc_copy_rows_if_batched(_p(flag), _p(gate), int(bool(invert)), _p(src), _l(lds * es), _l(rows * lds * es), _p(dst), _l(ldd * es),
                                            _l(rows * ldd * es), _l(rows), C * es, B, _S()), "uc_copy_rows_if_batched")
    return dst


def letterbox_u8(src, input_size, swap_rb=True, pad=114, out=None):
    """src: uint8 [h,w,3] device tensor (RGB when swap_rb) -> (uint8 [1,H,W,3] letterboxed frame, r) — the preprocessing of
    external/lib/test/tracker/unicorn_sot.py:114-123 (swap_rb=True) / data_augment.py:194-214 (swap_rb=False)."""
    assert src.dtype == torch.uint8 and src.is_cuda and src.is_contiguous() and src.dim() == 3 and src.shape[2] == 3
    h, w = src.shape[:2]
    H, W = input_size
    r = min(H / h, W / w)
    if out is None:
        out = torch.empty(1, H, W, 3, dtype=torch.uint8, device=src.device)
    _lib.check(_L().uc_letterbox_u8(_p(src), h, w, _p(out), H, W, int(h * r), int(w * r), int(bool(swap_rb)), int(pad), _S()), "uc_letterbox_u8")
    return out, r


def nchw_to_nhwc(x, dtype=torch.bfloat16, out=None):
    B, C, H, W = x.shape
    assert x.dtype == torch.float32 and x.is_contiguous()
    if out is None:
        out = torch.empty(B, H, W, C, dtype=dtype, device=x.device)
    _lib.check(_L().uc_nchw_f32_to_nhwc(_p(x), _p(out), _nhwc_ld(out), B, C, _l(H * W), _DT[out.dtype], _S()), "uc_nchw_f32_to_nhwc")
    return out


def nhwc_to_nchw(x):
    B, H, W, C = x.shape
    assert x.dtype in (torch.bfloat16, torch.float16), "uc_nhwc_to_nchw_f32 converts 16-bit NHWC maps"
    out = torch.empty(B, C, H, W, dtype=torch.float32, device=x.device)
    _lib.check(_L().uc_nhwc_to_nchw_f32(_p(x), _nhwc_ld(x), _p(out), B, C, _l(H * W), _DT[x.dtype], _S()), "uc_nhwc_to_nchw_f32")
    return out


def msda_forward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight):
    """Reference operator semantics (fp32)."""
    B, S, M, D = value.shape
    _, Lq, _, L, P, _ = sampling_loc.shape
    out = torch.empty(B, Lq, M * D, dtype=torch.float32, device=value.device)
    _lib.check(_L().uc_msda_forward_f32(_p(value), _p(spatial_shapes), _p(level_start_index), _p(sampling_loc), _p(attn_weight),
                                        B, S, M, D, L, Lq, P, _p(out), _S()), "uc_msda_forward_f32")
    return out


def msda_fused(value, offlog, level_hw, M=8, P=4, out=None):
    """value bf16 [B*Lq, M*32] with Lq = sum h*w over the levels: B images whose rows are level-major, the images inside each level
    (level l of image b at row B*start_l + b*h_l*w_l; B = 1 is the plain concatenation of the levels).  offlog and out: same rows."""
    L = len(level_hw)
    Lq = sum(h * w for h, w in level_hw)
    B = value.shape[0] // Lq
    assert value.shape == (B * Lq, M * 32) and B >= 1 and value.dtype == torch.bfloat16 and value.is_contiguous()
    assert offlog.dtype == torch.float32 and offlog.shape[0] == B * Lq and offlog.shape[1] >= M * L * P * 3
    if out is None:
        out = torch.empty(B * Lq, M * 32, dtype=torch.bfloat16, device=value.device)
    hw = (ctypes.c_int * (2 * L))(*[v for pair in level_hw for v in pair])
    if B == 1:
        _lib.check(_L().uc_msda_fused_bf16(_p(value), _p(offlog), offlog.stride(0), _p(out), hw, L, M, P, _S()), "uc_msda_fused_bf16")
    else:
        _lib.check(_L().uc_msda_fused_bf16_batched(_p(value), _p(offlog), offlog.stride(0), _p(out), hw, L, M, P, B, _S()),
                   "uc_msda_fused_bf16_batched")
    return out


def corr_propagate(embed_ref, embed_cur, values, out=None):
    """embed_* [n, 128] 16-bit rows; values fp32 [n_obj, n_ref] -> fp32 [n_obj, n_cur].  With a leading batch dimension (embed_*
    [B, n, 128], values [B, n_obj, n_ref], out [B, n_obj, n_cur]) the B sequences run in one launch, each as its own 2-D call."""
    if embed_ref.dim() == 2:
        n_ref, C = embed_ref.shape
        n_cur = embed_cur.shape[0]
        n_obj = values.shape[0]
        assert values.dtype == torch.float32 and values.stride(1) == 1 and values.shape[1] == n_ref
        if out is None:
            out = torch.empty(n_obj, n_cur, dtype=torch.float32, device=values.device)
        _lib.check(_L().uc_corr_propagate(_p(embed_ref), embed_ref.stride(0), n_ref, _p(embed_cur), embed_cur.stride(0), n_cur, C,
                                          _DT[embed_ref.dtype], _p(values), values.stride(0), n_obj, _p(out), out.stride(0), _S()),
                   "uc_corr_propagate")
        return out
    B, n_ref, C = embed_ref.shape
    n_cur = embed_cur.shape[1]
    n_obj = values.shape[1]
    assert embed_cur.shape[0] == B and values.shape[0] == B and values.shape[2] == n_ref
    assert values.dtype == torch.float32 and values.stride(2) == 1 and embed_ref.stride(2) == 1 and embed_cur.stride(2) == 1
    if out is None:
        out = torch.empty(B, n_obj, n_cur, dtype=torch.float32, device=values.device)
    assert out.shape == (B, n_obj, n_cur) and out.stride(2) == 1
    _lib.check(_L().uc_corr_propagate_batched(_p(embed_ref), embed_ref.stride(1), _l(embed_ref.stride(0)), n_ref, _p(embed_cur),
                                              embed_cur.stride(1), _l(embed_cur.stride(0)), n_cur, C, _DT[embed_ref.dtype], _p(values),
                                              values.stride(1), _l(values.stride(0)), n_obj, _p(out), out.stride(1), _l(out.stride(0)), B,
                                              _S()), "uc_corr_propagate_batched")
    return out


def head_decode(regobj, cls, hw, strides, ncls, out=None):
    """regobj / cls: 3 fp32 maps per level, rows [h*w, ld] of one image or NHWC [B,h,w,ld] of B images (image stride stride(0)).
    Returns fp32 [B, A, 5+ncls]."""
    A = sum(h * w for h, w in hw)
    B = regobj[0].shape[0] if regobj[0].dim() == 4 else 1
    if out is None:
        out = torch.empty(B, A, 5 + ncls, dtype=torch.float32, device=regobj[0].device)
    ro = (ctypes.c_void_p * 3)(*[t.data_ptr() for t in regobj])
    cl = (ctypes.c_void_p * 3)(*[t.data_ptr() for t in cls])
    hwa = (ctypes.c_int * 6)(*[v for pair in hw for v in pair])
    st = (ctypes.c_int * 3)(*strides)
    if B == 1:
        _lib.check(_L().uc_head_decode(ro, cl, hwa, st, regobj[0].shape[-1], cls[0].shape[-1], ncls, _p(out), _S()), "uc_head_decode")
        return out
    assert all(t.dim() == 4 and t.shape[0] == B for t in list(regobj) + list(cls)) and out.shape == (B, A, 5 + ncls) and out.is_contiguous()
    bs_ro = (ctypes.c_long * 3)(*[t.stride(0) for t in regobj])
    bs_cl = (ctypes.c_long * 3)(*[t.stride(0) for t in cls])
    _lib.check(_L().uc_head_decode_batched(ro, cl, hwa, st, regobj[0].shape[-1], cls[0].shape[-1], bs_ro, bs_cl, ncls, B, _p(out), _S()),
               "uc_head_decode_batched")
    return out


class PostWorkspace:
    """Device workspace and outputs of postprocess_device.  batch = 1: dets [A, 7], count [1], anchors [A]; batch = B > 1: one
    slice per image, dets [B, A, 7], count [B], anchors [B, A]."""

    def __init__(self, max_anchors, device, batch=1):
        fn = _L().uc_postprocess_workspace_bytes_batched
        fn.restype = ctypes.c_long
        self.nbytes = fn(max_anchors, batch)
        assert self.nbytes > 0, "PostWorkspace: batch must be >= 1"
        lead = (batch,) if batch > 1 else ()
        self.buf = torch.empty(self.nbytes, dtype=torch.uint8, device=device)
        self.dets = torch.empty(*lead, max_anchors, 7, dtype=torch.float32, device=device)
        self.count = torch.zeros(batch, dtype=torch.int32, device=device)
        self.anchors = torch.zeros(*lead, max_anchors, dtype=torch.int32, device=device)
        self.max_anchors, self.batch = max_anchors, batch


def postprocess_device(pred, ncls, conf, nms, ws, max_keep=0):
    """pred fp32 [A, 5+ncls] (decoded), or [B, A, 5+ncls] with a workspace of batch B.  Launches only; ws.dets / ws.count hold the
    result.  max_keep > 0 returns exactly the first max_keep rows of the full NMS result (per image)."""
    assert pred.is_contiguous() and pred.dtype == torch.float32 and pred.shape[-2] <= ws.max_anchors
    if pred.dim() == 3 and pred.shape[0] == 1:
        pred = pred[0]
    if pred.dim() == 2:
        A = pred.shape[0]
        _lib.check(_L().uc_postprocess(_p(pred), A, ncls, _f(conf), _f(nms), int(max_keep), _p(ws.buf), _l(ws.nbytes), _p(ws.dets), _p(ws.count), _p(ws.anchors), _S()),
                   "uc_postprocess", 4)
        return ws.dets, ws.count
    B, A = pred.shape[:2]
    assert B == ws.batch and A == ws.max_anchors, "postprocess_device: a batch of B images needs a PostWorkspace(A, device, batch=B)"
    _lib.check(_L().uc_postprocess_batched(_p(pred), A, ncls, _f(conf), _f(nms), int(max_keep), B, _p(ws.buf), _l(ws.nbytes), _p(ws.dets),
                                           _p(ws.count), _p(ws.anchors), _S()), "uc_postprocess_batched", 4)
    return ws.dets, ws.count


def sample_embed(embed, boxes, n_max, stride=8.0, count=None, out=None):
    """embed NHWC 16-bit [1,h,w,C]; boxes fp32 [>=n_max, >=4] (device); returns fp32 [n_max, C].
    B images: embed [B,h,w,C], boxes [B, >=n_max, >=4] (a batched PostWorkspace's dets), count int32 [B]; returns fp32 [B, n_max, C],
    image b sampling its own map at its own first min(count[b], n_max) boxes in one launch (the rows past that count are not written)."""
    B, h, w, C = embed.shape
    if boxes.dim() == 2:
        if out is None:
            out = torch.zeros(n_max, C, dtype=torch.float32, device=embed.device)
        _lib.check(_L().uc_sample_embed(_p(embed), _nhwc_ld(embed), h, w, C, _DT[embed.dtype], _p(boxes), boxes.stride(0), _p(count), n_max,
                                        _f(stride), _p(out), _S()), "uc_sample_embed")
        return out
    assert boxes.shape[0] == B and boxes.shape[1] >= n_max and boxes.stride(2) == 1 and count is not None and count.numel() == B
    if out is None:
        out = torch.zeros(B, n_max, C, dtype=torch.float32, device=embed.device)
    assert out.shape == (B, n_max, C) and out.dtype == torch.float32 and out.stride(2) == 1 and out.stride(1) == C
    if B == 1:
        _lib.check(_L().uc_sample_embed(_p(embed), _nhwc_ld(embed), h, w, C, _DT[embed.dtype], _p(boxes), boxes.stride(1), _p(count), n_max,
                                        _f(stride), _p(out), _S()), "uc_sample_embed")
        return out
    _lib.check(_L().uc_sample_embed_batched(_p(embed), _nhwc_ld(embed), _l(embed.stride(0)), h, w, C, _DT[embed.dtype], _p(boxes), boxes.stride(1),
                                            _l(boxes.stride(0)), _p(count), n_max, _f(stride), _p(out), _l(out.stride(0)), B, _S()),
               "uc_sample_embed_batched")
    return out


def bisoftmax(det_embeds, memo_embeds, det_labels=None, memo_labels=None):
    N, C = det_embeds.shape
    M = memo_embeds.shape[0]
    ws = torch.empty(N * M + 2 * N + 2 * M, dtype=torch.float32, device=det_embeds.device)
    scores = torch.empty(N, M, dtype=torch.float32, device=det_embeds.device)
    _lib.check(_L().uc_bisoftmax(_p(det_embeds), _p(memo_embeds), N, M, C, _p(det_labels), _p(memo_labels), _p(ws), _p(scores), _S()),
               "uc_bisoftmax", 3)
    return scores


def qd_assign(scores, memo_ids, boxes5, match_thr, obj_thr, nms_conf_thr):
    """scores f32 [N,M] (device), memo_ids int64 [M], boxes5 f32 [N,5] (score in column 4) -> ids int64 [N] (device)."""
    N, M = scores.shape
    ids = torch.full((N,), -1, dtype=torch.int64, device=boxes5.device)
    if N == 0:
        return ids
    taken = torch.empty(max(M, 1), dtype=torch.uint8, device=boxes5.device)
    _lib.check(_L().uc_qd_assign(_p(scores), N, M, _p(memo_ids), _p(boxes5[:, 4]), boxes5.stride(0), _f(match_thr), _f(obj_thr), _f(nms_conf_thr),
                                 _p(ids), _p(taken), _S()), "uc_qd_assign")
    return ids


def box_iou(a, b, plus_one=False):
    N, M = a.shape[0], b.shape[0]
    out = torch.empty(N, M, dtype=torch.float32, device=a.device)
    if N and M:
        _lib.check(_L().uc_box_iou(_p(a), a.stride(0), N, _p(b), b.stride(0), M, _p(out), int(plus_one), _S()), "uc_box_iou")
    return out


def aligned_bilinear_add(src, dst, factor):
    """dst += aligned_bilinear(src, factor) on NHWC bf16 maps [B,hs,ws,C] -> [B,hs*f,ws*f,C]; B > 1 images run in one launch."""
    B, hs, ws, C = src.shape
    assert dst.shape == (B, hs * factor, ws * factor, C)
    if B == 1:
        _lib.check(_L().uc_aligned_bilinear_add(_p(src), _nhwc_ld(src), hs, ws, _p(dst), _nhwc_ld(dst), C, factor, _S()), "uc_aligned_bilinear_add")
        return dst
    _lib.check(_L().uc_aligned_bilinear_add_batched(_p(src), _nhwc_ld(src), _l(src.stride(0)), hs, ws, _p(dst), _nhwc_ld(dst), _l(dst.stride(0)), C,
                                                    factor, B, _S()), "uc_aligned_bilinear_add_batched")
    return dst


def dynamic_masks(mask_feats, up_masks, dyn_levels, level_hw, ws, n_max, up_rate=4, d_rate=2, strides=(8, 16, 32), soi=(64.0, 128.0, 256.0),
                  out=None, scratch=None, image_of=None):
    """mask_feats fp32 [1,h,w,8]; up_masks fp32 [1,h,w,9*up^2]; dyn_levels: 3 fp32 [1,hk,wk,ld] controller outputs;
    ws: PostWorkspace after postprocess_device.  Returns fp32 [n_max, h*up*d, w*up*d].
    Batched: dyn_levels of B head images [B,hk,wk,ld], ws a PostWorkspace of batch B, and S mask-branch images (mask_feats
    [S,h,w,8], up_masks [S,h,w,9*up^2]); head image b reads mask-branch image image_of[b] (device int32 [B]; default b, with S = B)
    and an entry outside [0, S) skips it.  Returns fp32 [B, n_max, h*up*d, w*up*d]."""
    S, h, w, _ = mask_feats.shape
    B = dyn_levels[0].shape[0]
    H, W = h * up_rate * d_rate, w * up_rate * d_rate
    dl = (ctypes.c_void_p * 3)(*[t.data_ptr() for t in dyn_levels])
    hw = (ctypes.c_int * 6)(*[v for pair in level_hw for v in pair])
    st = (ctypes.c_int * 3)(*strides)
    so = (ctypes.c_float * 3)(*soi)
    if scratch is None:
        scratch = torch.empty(B * n_max * h * w * (1 + up_rate * up_rate), dtype=torch.float32, device=mask_feats.device)
    if B == 1 and image_of is None:
        if out is None:
            out = torch.zeros(n_max, H, W, dtype=torch.float32, device=mask_feats.device)
        _lib.check(_L().uc_dynamic_masks(_p(mask_feats), _p(up_masks), h, w, up_rate, d_rate, dl, dyn_levels[0].shape[-1], hw, st, so,
                                         _p(ws.anchors), _p(ws.count), n_max, _p(scratch), _p(out), _S()), "uc_dynamic_masks", 3)
        return out
    assert ws.batch == B and all(t.shape[0] == B and t.stride(-1) == 1 for t in dyn_levels), "dynamic_masks: B head images need a PostWorkspace of batch B"
    assert mask_feats.is_contiguous() and up_masks.is_contiguous() and up_masks.shape[0] == S
    assert scratch.numel() >= B * n_max * h * w * (1 + up_rate * up_rate)
    if image_of is None:
        assert S == B, "dynamic_masks: image_of is needed when the mask-branch images are not the head images"
        image_of = torch.arange(B, dtype=torch.int32, device=mask_feats.device)
    assert image_of.dtype == torch.int32 and image_of.numel() == B and image_of.is_contiguous()
    if out is None:
        out = torch.zeros(B, n_max, H, W, dtype=torch.float32, device=mask_feats.device)
    assert out.shape == (B, n_max, H, W) and out.is_contiguous()
    bs = (ctypes.c_long * 3)(*[t.stride(0) for t in dyn_levels])
    _lib.check(_L().uc_dynamic_masks_batched(_p(mask_feats), _p(up_masks), S, h, w, up_rate, d_rate, dl, dyn_levels[0].shape[-1], bs, hw, st, so,
                                             _p(ws.anchors), _l(ws.max_anchors), _p(ws.count), _p(image_of), B, n_max, _p(scratch), _p(out),
                                             _S()), "uc_dynamic_masks_batched", 3)
    return out


def vos_aggregate(masks, init_mask, ids, Hin, Win, r, soft, seg):
    """Result assembly of a VOS frame (uc_vos_aggregate): the soft masks of `ids` resized by 1/r to the original frame into soft fp32
    [>= n, H0, W0], and the label map seg uint8 [H0, W0] (argmax over the background product and the objects, in list order).
    masks: fp32 [1, Hin, Win] network-resolution masks of the first len(masks) ids; the remaining ids take (init_mask == id) of
    init_mask, a uint8 [H0, W0] label map."""
    objs, n, H0, W0 = _vos_objects(masks, init_mask, ids, Hin, Win, soft, seg)
    _lib.check(_L().uc_vos_aggregate(objs, n, Hin, Win, H0, W0, _f(r), _p(soft), _p(seg), _S()), "uc_vos_aggregate")
    return seg


def _vos_objects(masks, init_mask, ids, Hin, Win, soft, seg):
    """The host object array of one video of vos_aggregate (soft may be None), with its object count and original size."""
    n = len(ids)
    H0, W0 = seg.shape
    assert soft is None or (soft.dtype == torch.float32 and soft.is_contiguous() and soft.shape[0] >= n and tuple(soft.shape[1:]) == (H0, W0))
    assert seg.dtype == torch.uint8 and seg.is_contiguous() and len(masks) <= n
    objs = (_lib.UcVosObject * n)()
    for k, oid in enumerate(ids):
        objs[k].id = int(oid)
        if k < len(masks):
            assert masks[k].dtype == torch.float32 and masks[k].is_contiguous() and tuple(masks[k].shape[-2:]) == (Hin, Win)
            objs[k].mask = masks[k].data_ptr()
        else:
            assert init_mask is not None and init_mask.dtype == torch.uint8 and tuple(init_mask.shape) == (H0, W0)
            objs[k].init_mask = init_mask.data_ptr()
    return objs, n, H0, W0


def mots_encode_workspace(k_max, H, W, device):
    """Device workspace of uc_mots_encode for up to k_max instances on an H x W original frame."""
    fn = _L().uc_mots_encode_workspace_bytes
    fn.restype = ctypes.c_long
    return torch.empty(fn(int(k_max), int(H), int(W)), dtype=torch.uint8, device=device)


def mots_encode(masks, order, emit, thr, r, H, W, ws, chars, offsets, k=None):
    """COCO RLE strings of the resized, thresholded, overlap-free masks of one MOTS frame (uc_mots_encode).  masks fp32
    [n_max,Hin,Win]; order int32 [k] / emit uint8 [k] device; chars uint8 device buffer (its size is the capacity); offsets int64
    device [>= k+1].  Launches only: offsets[k] is the number of chars needed, chars past the capacity are not written.
    B images (uc_mots_encode_batched): masks [B,n_max,Hin,Win]; k, r, H, W: B instance counts, letterbox ratios and original sizes
    (host sequences); order / emit: the sum(k) entries of all images grouped by image (mask rows within the image's own block), and
    offsets [>= sum(k)+1] over all of them.  Each image's overlap removal is its own and its strings equal its one-image call's."""
    if masks.dim() == 3:
        n_max, Hin, Win = masks.shape
        k = order.numel()
        assert masks.dtype == torch.float32 and masks.is_contiguous() and order.dtype == torch.int32 and emit.dtype == torch.uint8
        assert emit.numel() == k and chars.dtype == torch.uint8 and offsets.dtype == torch.int64 and offsets.numel() >= k + 1
        _lib.check(_L().uc_mots_encode(_p(masks), n_max, Hin, Win, _p(order), _p(emit), k, _f(thr), ctypes.c_double(r), int(H), int(W),
                                       _p(ws), _l(ws.numel()), _p(chars), _l(chars.numel()), _p(offsets), _S()), "uc_mots_encode",
                   3 if k else 1)
        return offsets
    B, n_max, Hin, Win = masks.shape
    K = order.numel()
    assert masks.dtype == torch.float32 and masks.stride(3) == 1 and masks.stride(2) == Win and masks.stride(1) == Hin * Win
    assert k is not None and len(k) == len(r) == len(H) == len(W) == B and sum(k) == K
    assert order.dtype == torch.int32 and emit.dtype == torch.uint8 and emit.numel() == K
    assert chars.dtype == torch.uint8 and offsets.dtype == torch.int64 and offsets.numel() >= K + 1
    ints = lambda v: (ctypes.c_int * B)(*[int(x) for x in v])  # noqa: E731
    _lib.check(_L().uc_mots_encode_batched(_p(masks), _l(masks.stride(0)), n_max, Hin, Win, B, ints(k), ints(H), ints(W),
                                           (ctypes.c_double * B)(*[float(x) for x in r]), _p(order), _p(emit), _f(thr), _p(ws),
                                           _l(ws.numel()), _p(chars), _l(chars.numel()), _p(offsets), _S()), "uc_mots_encode_batched",
               3 if K else 1)
    return offsets

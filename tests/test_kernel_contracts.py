"""Argument validation of uc_groupnorm_apply, uc_copy_upsample, uc_add, uc_dwconv7_ln, uc_stem_ln and uc_conv2d: every call here is rejected with UC_EINVAL and a message
before anything is launched, so the pointers are fake addresses that are never dereferenced and the test runs without a GPU."""
import ctypes

import pytest

from unicorn_b200 import _lib

P = ctypes.c_void_p
EINVAL = -1
A16 = [P(0x10000 * (i + 1)) for i in range(6)]  # 16-byte aligned, never dereferenced


@pytest.fixture(scope="module")
def lib():
    return _lib.lib()


def gn(lib, x=A16[0], ldx=256, stats=A16[1], w=A16[2], b=A16[3], y=A16[4], ldy=256, B=1, HW=16, C=256, G=16, eps=1e-3,
       act=_lib.ACT_SILU, prior=None, beta=None, add2=None, ldadd2=0, y2=None, ldy2=0):
    rc = lib.uc_groupnorm_apply(x, ldx, stats, w, b, y, ldy, B, ctypes.c_long(HW), C, G, ctypes.c_float(eps), act, prior, beta, add2,
                                ldadd2, y2, ldy2, None)
    return rc, lib.uc_last_error()


def rejected(call, *words):
    rc, msg = call
    assert rc == EINVAL, (rc, msg)
    for w in words:
        assert w.encode() in msg, (w, msg)


@pytest.mark.parametrize("act", [_lib.ACT_GELU, _lib.ACT_SIGMOID, 5, -1])
def test_groupnorm_apply_rejects_activations_it_does_not_implement(lib, act):
    rejected(gn(lib, act=act), "uc_groupnorm_apply", "act must be")


def test_groupnorm_apply_rejects_bad_groups_and_sizes(lib):
    rejected(gn(lib, G=0), "G must be >= 1")  # used to divide by zero (SIGFPE) in the host process
    rejected(gn(lib, G=-16), "G must be >= 1")
    rejected(gn(lib, G=24), "C % G == 0")
    rejected(gn(lib, C=252, ldx=256, ldy=256), "multiples of 8")
    rejected(gn(lib, ldx=260), "multiples of 8")
    rejected(gn(lib, C=4104, G=8, ldx=4104, ldy=4104), "C too large")
    rejected(gn(lib, C=4104, G=8, ldx=4104, ldy=4104, x=None, stats=None, w=None, b=None, y=None), "C too large")
    # C = 4096 is accepted: with null pointers the call gets past the size checks and stops at the pointer check
    rejected(gn(lib, C=4096, G=32, ldx=4096, ldy=4096, x=None, stats=None, w=None, b=None, y=None), "null pointer")


def test_groupnorm_apply_rejects_bad_pointers(lib):
    rejected(gn(lib, x=None), "null pointer")
    rejected(gn(lib, prior=A16[5]), "prior and beta go together")
    rejected(gn(lib, y2=A16[5]), "bad second output")
    for k in ("x", "y"):
        rejected(gn(lib, **{k: P(0x10008)}), "16-byte aligned")
    # a channel slice 4 bf16 elements into a 16-byte aligned buffer: legal strides, misaligned base
    rejected(gn(lib, x=P(0x10008), y=P(0x10008)), "16-byte aligned")
    rejected(gn(lib, add2=P(0x50008), ldadd2=256, y2=A16[5], ldy2=256), "16-byte aligned")
    rejected(gn(lib, add2=A16[5], ldadd2=256, y2=P(0x60004), ldy2=256), "16-byte aligned")
    rejected(gn(lib, stats=P(0x20004)), "stats must be 8-byte aligned")


def test_copy_upsample_rejects_misaligned_maps(lib):
    cu = lambda src, dst, up=2, C=64: (lib.uc_copy_upsample(src, 64, dst, 160, 1, 4, 4, C, up, None), lib.uc_last_error())  # noqa: E731
    rejected(cu(P(0x10008), A16[1]), "uc_copy_upsample", "16-byte aligned")
    rejected(cu(A16[0], P(0x20008)), "uc_copy_upsample", "16-byte aligned")
    rejected(cu(A16[0], A16[1], up=3), "uc_copy_upsample: bad arguments")
    rejected(cu(A16[0], A16[1], C=60), "uc_copy_upsample: bad arguments")
    rejected(cu(None, A16[1]), "uc_copy_upsample: bad arguments")


def test_add_rejects_misaligned_rows_and_other_dtypes(lib):
    add = lambda a, b, y, dtype=_lib.BF16: (lib.uc_add(a, 64, b, 64, y, 64, ctypes.c_long(10), 64, dtype, None), lib.uc_last_error())  # noqa: E731
    for args in ((P(0x10008), A16[1], A16[2]), (A16[0], P(0x20008), A16[2]), (A16[0], A16[1], P(0x30004))):
        rejected(add(*args), "uc_add", "16-byte aligned")
    rejected(add(A16[0], A16[1], A16[2], dtype=_lib.F32), "uc_add", "16-bit dtypes only")
    rejected(add(A16[0], None, A16[2]), "uc_add: bad arguments")


def dwln(lib, x=A16[0], w=A16[1], bias=A16[2], lnw=A16[3], lnb=A16[4], y=A16[5], B=1, H=8, W=8, C=128):
    rc = lib.uc_dwconv7_ln(x, w, bias, lnw, lnb, y, B, H, W, C, ctypes.c_float(1e-6), None)
    return rc, lib.uc_last_error()


def test_dwconv7_ln_rejects_bad_channels_in_place_and_null(lib):
    for C in (127, 1, 1538, 2048, 0):
        rejected(dwln(lib, C=C), "uc_dwconv7_ln", "C must be even and <= 1536")
    rejected(dwln(lib, y=A16[0]), "uc_dwconv7_ln", "not an in-place operation")
    for k in ("x", "w", "bias", "lnw", "lnb", "y"):
        rejected(dwln(lib, **{k: None}), "uc_dwconv7_ln", "null pointer")


def stem(lib, img=A16[0], w=A16[1], bias=A16[2], lnw=A16[3], lnb=A16[4], out=A16[5], B=1, H=32, W=32, C0=96):
    rc = lib.uc_stem_ln(img, 0, w, bias, lnw, lnb, out, B, H, W, C0, ctypes.c_float(1e-6), None)
    return rc, lib.uc_last_error()


def test_stem_ln_rejects_bad_shapes_channels_and_null(lib):
    for H, W in ((30, 32), (32, 34), (2, 32)):
        rejected(stem(lib, H=H, W=W), "uc_stem_ln", "H%4==0, W%4==0")
    rejected(stem(lib, C0=288), "uc_stem_ln", "C0<=256")
    rejected(stem(lib, C0=100), "uc_stem_ln", "C0%32==0")
    rejected(stem(lib, C0=160), "uc_stem_ln: unsupported C0 160")  # 5 channels per lane: no kernel instantiated
    rejected(stem(lib, C0=224), "uc_stem_ln: unsupported C0 224")
    for k in ("img", "w", "bias", "lnw", "lnb", "out"):
        rejected(stem(lib, **{k: None}), "uc_stem_ln", "null pointer")


def conv(lib, **kw):
    """uc_conv2d on a valid 3x3 / s1 / p1 bf16 conv of 1 x 16 x 16 x 64 -> 64 channels, with the fields in kw replaced."""
    d = _lib.UcConv2d()
    d.x, d.x_dtype, d.B, d.H, d.W, d.Cin, d.ldx = A16[0], _lib.BF16, 1, 16, 16, 64, 64
    d.w, d.Cout, d.KH, d.KW, d.stride, d.pad = A16[1], 64, 3, 3, 1, 1
    d.y, d.ldy, d.y_dtype, d.act = A16[2], 64, _lib.BF16, _lib.ACT_NONE
    for k, v in kw.items():
        setattr(d, k, v)
    rc = lib.uc_conv2d(ctypes.byref(d), None)
    return rc, lib.uc_last_error()


def test_conv2d_rejects_empty_maps(lib):
    for k in ("B", "H", "W"):
        for v in (0, -1):
            rejected(conv(lib, **{k: v}), "uc_conv2d: B, H and W must be >= 1")


@pytest.mark.parametrize("KH,KW,stride,pad,H,W", [
    (3, 3, 1, 0, 2, 16), (3, 3, 1, 0, 16, 2), (3, 1, 1, 0, 1, 16),   # stride 1: (H + 2 pad - KH) = -1
    (2, 2, 2, 0, 1, 16), (2, 2, 2, 0, 16, 1),                        # stride 2, numerator -1: C's division gave an output of 1
    (3, 3, 2, 0, 2, 16), (3, 3, 2, 0, 16, 2), (3, 3, 2, 0, 1, 1)])
def test_conv2d_rejects_kernels_larger_than_the_padded_map(lib, KH, KW, stride, pad, H, W):
    rejected(conv(lib, KH=KH, KW=KW, stride=stride, pad=pad, H=H, W=W), "uc_conv2d", "kernel larger than the padded map")


def test_conv2d_rejects_a_conv_that_reads_only_padding(lib):
    # 1x1 / s2 / p1 on a map one pixel high (wide): every tap falls on the empty odd phase, the output would be the bias alone
    rejected(conv(lib, KH=1, KW=1, stride=2, pad=1, H=1, W=16), "uc_conv2d", "reads only zero padding")
    rejected(conv(lib, KH=3, KW=1, stride=2, pad=1, H=5, W=1), "uc_conv2d", "reads only zero padding")


def test_conv2d_rejects_bad_groupnorm_tiles(lib):
    st = A16[3]
    rejected(conv(lib, gn_stats=st, gn_groups=24), "uc_conv2d: bad GroupNorm grouping")  # 24 does not divide 64
    rejected(conv(lib, gn_stats=st, gn_groups=0), "uc_conv2d: bad GroupNorm grouping")
    rejected(conv(lib, gn_stats=st, gn_groups=-8), "uc_conv2d: bad GroupNorm grouping")
    # group size 24 (Cout 192, 8 groups) straddles a 64-column N tile
    rejected(conv(lib, Cout=192, ldy=192, gn_stats=st, gn_groups=8, block_n=64), "N tile 64 incompatible with GroupNorm group size 24")
    rejected(conv(lib, Cout=192, ldy=192, gn_stats=st, gn_groups=8, block_n=1256), "N tile 256 incompatible with GroupNorm group size 24")
    # group size 5 or 25: no N tile is a multiple of it, so the heuristic (block_n = 0) has nothing to pick
    rejected(conv(lib, Cout=40, ldy=40, gn_stats=st, gn_groups=8), "no N tile compatible with GroupNorm group size 5")
    rejected(conv(lib, Cout=200, ldy=200, gn_stats=st, gn_groups=8), "no N tile compatible with GroupNorm group size 25")
    # a CTA accumulates at most 64 groups: group size 1 or 2 at wide N tiles
    for bn, gs in ((96, 1), (128, 1), (256, 2), (192, 2), (1128, 1), (1256, 2)):
        rejected(conv(lib, Cout=256, ldy=256, gn_stats=st, gn_groups=256 // gs, block_n=bn), f"uc_conv2d: N tile {bn % 1000} holds "
                 f"{bn % 1000 // gs} GroupNorm groups, more than the 64")


@pytest.mark.parametrize("block_n", [1064, 1096, 1016, 1000, 2256])
def test_conv2d_rejects_cluster_block_n_without_a_cluster_variant(lib, block_n):
    rejected(conv(lib, block_n=block_n), "uc_conv2d: the cluster variant exists for block_n 128/192/256 only")


@pytest.mark.parametrize("block_n", [8, 48, 100, 112, 160, 512, 999, -16])
def test_conv2d_rejects_unsupported_block_n(lib, block_n):
    rejected(conv(lib, block_n=block_n), f"uc_conv2d: unsupported block_n {block_n}")


def test_conv2d_rejects_act_after_res_combinations(lib):
    r = dict(res=A16[4], ldres=64, act=_lib.ACT_RELU, act_after_res=1)
    msg = "uc_conv2d: act_after_res needs act = ReLU, res and bf16 x"
    for bad in (dict(act=_lib.ACT_NONE), dict(act=_lib.ACT_GELU), dict(res=None), dict(x_dtype=_lib.F16, y_dtype=_lib.F16),
                dict(gamma=A16[5]), dict(gn_stats=A16[3], gn_groups=16), dict(row_stats=A16[3], col_s=A16[5], KH=1, KW=1, pad=0)):
        rejected(conv(lib, **{**r, **bad}), msg)


def test_conv2d_rejects_row_stats_off_a_flat_conv(lib):
    ln = dict(row_stats=A16[3], col_s=A16[5], act=_lib.ACT_GELU)
    msg = "uc_conv2d: row_stats (folded LayerNorm) needs a 1x1 stride-1 conv and col_s"
    rejected(conv(lib, **ln), msg)  # 3x3
    rejected(conv(lib, **ln, KH=1, KW=1, pad=0, stride=2), msg)
    rejected(conv(lib, **ln, KH=1, KW=1, pad=1), msg)
    rejected(conv(lib, **{**ln, "col_s": None}, KH=1, KW=1, pad=0), msg)

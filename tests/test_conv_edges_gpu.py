"""uc_conv2d (the implicit-GEMM convolution, conv_gemm.cuh) bit for bit on exact operands and per element against float64.

Exact lattice: x and w are integers in [-3, 3] (exact in bf16 and f16) and S = conv(|x|, |w|) < 2^20 at every output (asserted),
so every partial sum of the fp32 wgmma accumulator is an exact integer in any order and the accumulator equals the float64
convolution.  The epilogue is then emulated in float32 in the kernel's order (conv_gemm.cuh, the consumers' epilogue loop):
pre = f32(acc + bias); act (ReLU exact); y = f32(y * gamma) (__fmul_rn; gamma is 1.0 when absent); y = f32(y + res);
ReLU after the residual; round to nearest even to bf16 / f16 (fp32 y is stored unrounded).  Each step rounds once and torch's
float32 ops round the same way, so bias, gamma and the residual can be arbitrary and the output must be equal bit for bit.
GELU, SiLU and sigmoid are fits: their outputs must lie within one ulp (plus the fit error) of the float64 activation.

GroupNorm statistics on the lattice: a bias that is a multiple of 1/8 and |pre| <= 8 (asserted) keep every fp32 partial sum of
pre and pre^2 exact, so the int64 statistics must be 2^22 sum(pre) and 2^22 sum(pre^2) exactly.

Production magnitudes: Gaussian operands at the real K; per element, the bound is one rounding of the output (2^-8 |ref| for
bf16) + |gamma| K u S (the fp32 GEMM: exact products, at most one rounding per accumulation step) + 2^-22 (|res| + |gamma pre|)
for the epilogue + a small floor.  Every check prints its largest err / bound."""
import math

import pytest
import torch
import torch.nn.functional as F

from unicorn_b200 import ops
from unicorn_b200._lib import UnicornB200Error

pytestmark = pytest.mark.gpu
dev = "cuda"
U = 2.0 ** -24   # fp32 unit roundoff
FIX = 2.0 ** 22  # fixed-point scale of the GroupNorm statistics (kGnFixedScale)
GELU_FIT = 4e-6  # |GELU fit - erf GELU| over the real line (test_gelu_fit.py)
ACT_LIP = 1.13   # max |GELU'| = 1.1289; SiLU' <= 1.1, sigmoid' <= 0.25
REL = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11, torch.float32: U}  # one rounding of the output
BLOCK_NS = (16, 32, 64, 96, 128, 192, 256, 1128, 1192, 1256)
EDGE_CIN = (8, 24, 56, 64, 72, 136, 200)  # the last 64-channel chunk partial (or the only one)
ACTS = {"none": ops.ACT_NONE, "relu": ops.ACT_RELU, "gelu": ops.ACT_GELU, "silu": ops.ACT_SILU, "sigmoid": ops.ACT_SIGMOID}


def G(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def check(got, ref, bound, name):
    """Per-element |got - ref| <= bound; ref and bound float64."""
    err = (got.double() - ref).abs()
    ratio = (err / bound).max().item()
    print(f"err/bound {ratio:.3f}  {name}")
    assert ratio <= 1.0, f"{name}: max err/bound {ratio:.3g} (max err {err.max().item():.3g})"
    return ratio


def ulp(v, dtype):
    """Spacing of the bf16 / f16 numbers at |v| (normal range)."""
    _, e = torch.frexp(v.abs())
    return torch.ldexp(torch.ones_like(v), e - (8 if dtype == torch.bfloat16 else 11))


def nchw(t):
    return t.permute(0, 3, 1, 2)


def nhwc(t):
    return t.permute(0, 2, 3, 1)


def unpack(wp, Cout, KH, KW):
    """[Cout_pad, KH*KW, Cin] packed weights -> float64 [Cout, Cin, KH, KW]."""
    return wp[:Cout].double().reshape(Cout, KH, KW, -1).permute(0, 3, 1, 2)


def conv64(x, w, stride, pad):
    return nhwc(F.conv2d(nchw(x.double()), w, stride=stride, padding=pad))


# ---------------------------------------------------------------------------------------------------------------- mirrors
def tile_w(Wo, Ho):
    """The output tile uc_conv2d picks (conv_gemm.cu): the tile_w x 128 / tile_w patch with the fewest tiles, widest on ties."""
    best, bw = None, 128
    for tw in (128, 64, 32, 16, 8):
        n = -(-Wo // tw) * -(-Ho // (128 // tw))
        if best is None or n < best:
            best, bw = n, tw
    return bw


def out_hw(H, W, KH, KW, s, pad):
    if KH == 1 and KW == 1 and s == 1 and pad == 0:
        return 1, H * W  # a flat conv is one row of H * W pixels per image
    return (H + 2 * pad - KH) // s + 1, (W + 2 * pad - KW) // s + 1


def epi_variant(x_dtype, y_dtype, act, gamma=False, res=False, gn=False, act_after_res=False):
    """The epilogue instantiation uc_conv2d dispatches to (conv_gemm.cu; no folded LayerNorm here)."""
    if x_dtype == torch.float16:
        return "any"
    bf16y = y_dtype == torch.bfloat16
    if act_after_res:
        return "relu_res" if bf16y else "any"
    if res:
        return "res" if bf16y and act == "none" and not gn else "any"
    if gn:
        return "gn" if bf16y and act == "none" and not gamma else "any"
    if gamma:
        return "any"
    if y_dtype == torch.float32:
        return "f32" if act == "none" else "any"
    if y_dtype == torch.float16:
        return "bias_f16" if act == "none" else "any"
    return {"none": "bias", "relu": "relu", "gelu": "gelu"}.get(act, "any")


VARIANTS = {"bias", "bias_f16", "f32", "relu", "gelu", "res", "relu_res", "gn", "any"}


# ---------------------------------------------------------------------------------------------------------------- lattice
def lattice(shape, g, lo=-3, hi=3):
    return torch.randint(lo, hi + 1, shape, generator=g).double()


def emulate(acc, bias, act="none", gamma=None, res=None, act_after_res=False, out_dtype=torch.bfloat16, alt=None):
    """The epilogue in float32 in the kernel's order on the exact accumulator acc (float64 integers).  alt selects a wrong
    rounding point: "pre_bf16" (pre rounded to bf16 before the residual add), "fma" (y * gamma + res with one rounding),
    "rtz" (round-toward-zero packing to bf16)."""
    y = acc.float()
    if bias is not None:
        y = y + bias
    if act == "relu" and not act_after_res:
        y = torch.relu(y)
    if alt == "pre_bf16":
        y = y.bfloat16().float()
    if alt == "fma" and gamma is not None and res is not None:
        y = (y.double() * gamma.double() + res.double()).float()
    else:
        if gamma is not None:
            y = y * gamma
        if res is not None:
            y = y + res.float()
    if act_after_res:
        y = torch.relu(y)
    if alt == "rtz":
        return (y.view(torch.int32) & -65536).view(torch.float32).bfloat16()
    return y.to(out_dtype)


def act64(z, act):
    if act == "gelu":
        return 0.5 * z * (1 + torch.erf(z / math.sqrt(2)))
    if act == "silu":
        return z * torch.sigmoid(z)
    if act == "sigmoid":
        return torch.sigmoid(z)
    return torch.relu(z) if act == "relu" else z


def channel_slice(t, lead, extra, g):
    """t inside a wider, randomly filled buffer: channels [lead, lead + C) of rows of C + extra elements (ld > C), plus a guard
    image after the B images.  Returns (view, buffer)."""
    B, H, W, C = t.shape
    buf = torch.randn(B + 1, H, W, C + extra, generator=g).to(dev).to(t.dtype)
    view = buf[:B, :, :, lead:lead + C]
    view.copy_(t)
    return view, buf


def run_lattice(B, H, W, Cin, Cout, KH, KW, stride, pad, seed, x_dtype=torch.bfloat16, out_dtype=torch.bfloat16, act="none",
                gamma=False, res=False, act_after_res=False, gn=0, block_n=0, slices=False, in_place=False, bias=True, alts=()):
    """One lattice launch, compared bit for bit with the emulated epilogue.  slices: x, y (and res) are channel slices of wider
    buffers with guard columns and a guard image, all of which must stay unchanged; in_place: the residual is y itself.
    Returns (variant, out, y before packing for the tie count, {alt: number of outputs that differ})."""
    g = G(seed)
    x = lattice((B, H, W, Cin), g).to(dev).to(x_dtype)
    w = lattice((Cout, Cin, KH, KW), g)
    wp = ops.pack_conv_weight(w.float().to(dev), x_dtype)
    Ho, Wo = (H + 2 * pad - KH) // stride + 1, (W + 2 * pad - KW) // stride + 1
    acc = conv64(x, w.to(dev), stride, pad)
    S = conv64(x.abs(), w.abs().to(dev), stride, pad)
    assert S.max().item() < 2 ** 20, "lattice premise: partial sums below 2^20"
    b = torch.randn(Cout, generator=g).to(dev) if bias else None
    gm = (0.5 * torch.randn(Cout, generator=g)).to(dev) if gamma else None
    r = torch.randn(B, Ho, Wo, Cout, generator=g).to(dev).to(out_dtype) if res or act_after_res else None
    kw = dict(bias=b, act=ACTS[act], gamma=gm, block_n=block_n, act_after_res=act_after_res)
    xs, guards = x, []
    if gn:
        stbuf = torch.zeros(B + 1, gn, 2, dtype=torch.int64, device=dev)  # a guard image after the statistics
        kw.update(gn_stats=stbuf[:B], gn_groups=gn)
        guards.append((stbuf[B], stbuf[B].clone(), "statistics guard image"))
    if slices:
        xs, xbuf = channel_slice(x, 8, 24, g)
        guards.append((xbuf, xbuf.clone(), "x buffer"))
    ybuf = torch.randn(B + 1, Ho, Wo, Cout + (16 if slices else 0), generator=g).to(dev).to(out_dtype)
    y = ybuf[:B, :, :, 8:8 + Cout] if slices else ybuf[:B]
    if r is not None:
        if in_place:
            y.copy_(r)
            kw["res"] = y
        elif slices:
            rs, rbuf = channel_slice(r, 16, 32, g)
            kw["res"] = rs
            guards.append((rbuf, rbuf.clone(), "residual buffer"))
        else:
            kw["res"] = r.clone()
    ybuf0 = ybuf.clone()
    out = ops.conv2d(xs, wp, KH, KW, stride, pad, out=y, **kw)
    torch.cuda.synchronize()
    tag = f"B={B} H={H} W={W} Cin={Cin} Cout={Cout} {KH}x{KW}/s{stride}/p{pad} bn={block_n} act={act} out={out_dtype}"
    for buf, buf0, what in guards:
        assert torch.equal(buf, buf0), f"{tag}: {what} changed"
    mask = torch.ones_like(ybuf, dtype=torch.bool)
    if slices:
        mask[:B, :, :, 8:8 + Cout] = False
    else:
        mask[:B] = False
    assert torch.equal(ybuf[mask], ybuf0[mask]), f"{tag}: guard columns or guard image of the output changed"
    variant = epi_variant(x_dtype, out_dtype, act, gamma, r is not None, gn > 0, act_after_res)
    ref_kw = dict(act=act, gamma=gm, res=r, act_after_res=act_after_res)
    if act in ("gelu", "silu", "sigmoid"):
        assert gm is None and r is None, "the fitted activations are checked without gamma and residual"
        pre = acc + b.double() if b is not None else acc
        ref = act64(pre, act)
        # one rounding of the kernel's fp32 value: at most one ulp of ref, also where that value and ref lie on either side of a
        # power of two; the fit (ex2 / rcp approximations for SiLU and sigmoid: 2^-20 relative); the fp32 rounding of pre through
        # |act'| <= 1.13
        fit = GELU_FIT if act == "gelu" else 2.0 ** -20 * ref.abs() + 1e-7
        bound = ulp(ref, out_dtype) + fit + ACT_LIP * U * pre.abs()
        check(out, ref, bound, f"lattice [{variant}] {tag}")
        return variant, out, None, {}
    want = emulate(acc, b, out_dtype=out_dtype, **ref_kw)
    if not torch.equal(out, want):
        bad = (out != want).nonzero()
        i = tuple(bad[0].tolist())
        raise AssertionError(f"lattice [{variant}] {tag}: {bad.shape[0]} of {out.numel()} outputs differ, first {i}: got "
                             f"{out[i].item()} want {want[i].item()} (acc {acc[i].item()})")
    diffs = {a: int((emulate(acc, b, out_dtype=out_dtype, alt=a, **ref_kw) != out).sum().item()) for a in alts}
    ypre = emulate(acc, b, out_dtype=torch.float32, **ref_kw)
    return variant, out, ypre, diffs


def report_bitwise(results, name):
    """Prints how many outputs of how many launches were compared bit for bit (the fitted activations are bounded instead)."""
    exact = [out.numel() for _, out, ypre, _ in results if ypre is not None]
    print(f"bitwise: {sum(exact)} outputs of {len(exact)} launches equal  {name}")


# name: (keywords of run_lattice).  Every epilogue variant, kEpiAny through each of the combinations it alone covers.
CONFIGS = {
    "bias": dict(),
    "no_bias": dict(bias=False),
    "bias_f16out": dict(out_dtype=torch.float16),
    "f32out": dict(out_dtype=torch.float32),
    "relu": dict(act="relu"),
    "gelu": dict(act="gelu"),
    "res": dict(res=True),
    "res_gamma": dict(res=True, gamma=True),
    "relu_res": dict(act="relu", act_after_res=True),
    "gn": dict(gn=50),  # with Cout 200: group size 4, which every N tile takes
    "any_f16x": dict(x_dtype=torch.float16, out_dtype=torch.float16, act="relu", gamma=True, res=True),
    "any_f16x_f32out": dict(x_dtype=torch.float16, out_dtype=torch.float32),
    "any_gamma_only": dict(gamma=True),
    "any_f16res": dict(out_dtype=torch.float16, gamma=True, res=True),
    "any_relu_res_f16out": dict(out_dtype=torch.float16, act="relu", act_after_res=True),
    "any_relu_f32out": dict(out_dtype=torch.float32, act="relu"),
    "any_relu_gn": dict(act="relu", gn=50),
    "any_silu": dict(act="silu"),
    "any_sigmoid": dict(act="sigmoid"),
}
LATTICE_COUT = (8, 24, 136, 200, 264)


def config_variant(name):
    c = CONFIGS[name]
    return epi_variant(c.get("x_dtype", torch.bfloat16), c.get("out_dtype", torch.bfloat16), c.get("act", "none"),
                       c.get("gamma", False), c.get("res", False) or c.get("act_after_res", False), bool(c.get("gn")),
                       c.get("act_after_res", False))


def test_configs_reach_every_epilogue_variant():
    hit = {config_variant(n) for n in CONFIGS}
    assert hit == VARIANTS, hit


@pytest.mark.parametrize("block_n", BLOCK_NS)
@pytest.mark.parametrize("name", list(CONFIGS))
def test_lattice_epilogues_bitwise(name, block_n):
    """Every epilogue variant at every N tile, bit for bit: a flat conv of 3 images of 7 x 45 pixels (3 partial 128-pixel tiles
    each, 9 M tiles: the cluster variant's padding tile) and a 3x3 / s1 / p1 conv of 2 images of 13 x 21, at Cout values that
    leave partial N tiles, Cin 72 (a partial 64-channel chunk)."""
    c = CONFIGS[name]
    i = list(CONFIGS).index(name)
    results = []
    for j, (B, H, W, K, pad) in enumerate(((3, 7, 45, 1, 0), (2, 13, 21, 3, 1))):
        Cout = 200 if c.get("gn") else LATTICE_COUT[(i + j + BLOCK_NS.index(block_n)) % len(LATTICE_COUT)]
        results.append(run_lattice(B, H, W, 72, Cout, K, K, 1, pad, 1000 * i + 10 * j + block_n, block_n=block_n, **c))
        assert results[-1][0] == config_variant(name)
    report_bitwise(results, f"[{config_variant(name)}] {name} bn={block_n}")


def test_rounding_points_are_pinned():
    """The kernel's output equals the emulation and differs, on the same operands, from each alternative ordering: pre rounded
    to bf16 before the residual add, an FMA-contracted y * gamma + res, and round-toward-zero packing.  The outputs include exact
    bf16 ties (fp32 values halfway between two bf16 numbers), so round-to-nearest-even is exercised."""
    alts = ("pre_bf16", "fma", "rtz")
    # an FMA changes the fp32 sum by at most one ulp, which shows in bf16 only next to a rounding tie: 2^16 pixels x 264 channels
    r1 = run_lattice(2, 128, 256, 72, 264, 1, 1, 1, 0, 7, res=True, gamma=True, alts=alts)
    r2 = run_lattice(3, 17, 45, 200, 136, 3, 3, 1, 1, 8, bias=False, alts=("rtz",))
    report_bitwise([r1, r2], "rounding points")
    d, (_, out, ypre, d2) = r1[3], r2
    ties = int(((ypre.view(torch.int32) & 0xFFFF) == 0x8000).sum().item())
    print(f"rounding points: outputs differing from the alternatives {d} (res + gamma), {d2} (no bias); {ties} exact bf16 ties "
          f"among {out.numel()} outputs")
    for a in alts:
        assert d[a] > 0, f"alternative {a} agrees with the kernel on every output: the check would not see it"
    assert d2["rtz"] > 0 and ties > 0


# ---------------------------------------------------------------------------------------------------------------- geometry
FILTERS = [(1, 1, 1, 0), (1, 1, 2, 0), (2, 2, 2, 0), (3, 3, 1, 1), (3, 3, 2, 1), (3, 3, 1, 0)]  # KH, KW, stride, pad


def geometry_maps():
    """(B, H, W) per filter: maps whose output selects each tile_w, +-1 around their seams, maps smaller than a tile, odd sizes
    at stride 2, and flat convs with B > 1 and H * W not a multiple of 128."""
    outs = [(64, 8), (40, 16), (20, 32), (6, 64), (3, 120), (65, 9), (39, 15), (21, 33), (7, 63), (2, 129), (1, 1), (3, 5), (5, 3)]
    maps = []
    for KH, KW, s, pad in FILTERS:
        for i, (Ho, Wo) in enumerate(outs):
            H, W = (Ho - 1) * s + KH - 2 * pad, (Wo - 1) * s + KW - 2 * pad
            if s == 2 and i % 2:
                H, W = H + 1, W + 1  # odd sizes / one row and column that no tap reaches
            maps.append((KH, KW, s, pad, 2 if i % 3 == 0 else 1, max(H, 1), max(W, 1)))
    maps += [(1, 1, 1, 0, 3, 7, 45), (1, 1, 1, 0, 2, 9, 15), (1, 1, 1, 0, 4, 1, 1), (1, 1, 1, 0, 3, 11, 23)]
    return maps


def test_geometry_maps_hit_every_tile_shape():
    hit = {tile_w(*reversed(out_hw(H, W, KH, KW, s, pad))) for KH, KW, s, pad, B, H, W in geometry_maps()}
    assert hit == {8, 16, 32, 64, 128}, hit


@pytest.mark.parametrize("Cin", EDGE_CIN)
def test_lattice_geometry_bitwise(Cin):
    """Every filter of FILTERS on every map of geometry_maps, x, y and the residual as channel slices with guards (in place for
    every third map), bit for bit."""
    tiles, results = set(), []
    for i, (KH, KW, s, pad, B, H, W) in enumerate(geometry_maps()):
        Cout = LATTICE_COUT[i % len(LATTICE_COUT)]
        results += [run_lattice(B, H, W, Cin, Cout, KH, KW, s, pad, 100 * Cin + i, res=True, gamma=i % 2 == 0, slices=True,
                    in_place=i % 3 == 0, block_n=(0, 16, 64, 1128)[i % 4])]
        tiles.add(tile_w(*reversed(out_hw(H, W, KH, KW, s, pad))))
    assert tiles == {8, 16, 32, 64, 128}
    report_bitwise(results, f"geometry Cin={Cin}")


@pytest.mark.parametrize("stride", [1, 2])
def test_lattice_every_filter_shape(stride):
    """Every (KH, KW) with at most 9 taps and every pad <= KH the entry point accepts, on a 2 x 11 x 13 map, bit for bit."""
    results = []
    for KH in range(1, 10):
        for KW in range(1, 10):
            if KH * KW > 9:
                continue
            for pad in range(KH + 1):
                if 11 + 2 * pad < KH or 13 + 2 * pad < KW:
                    continue
                results.append(run_lattice(2, 11, 13, 72, 24, KH, KW, stride, pad, 7000 + 100 * KH + 10 * KW + pad, res=True))
    report_bitwise(results, f"{len(results)} filter shapes at stride {stride}")


@pytest.mark.parametrize("KH,KW,pad,H,W", [(3, 3, 1, 1, 1), (3, 3, 1, 9, 1), (3, 3, 1, 1, 9), (3, 3, 1, 1, 130), (2, 2, 1, 1, 5),
                                           (1, 3, 0, 1, 9), (3, 1, 0, 9, 1), (1, 1, 0, 1, 9), (3, 3, 2, 1, 1)])
def test_stride2_one_pixel_maps_lattice(KH, KW, pad, H, W):
    """Stride 2 on a map one pixel high or wide: the odd stride phase has no pixels, and the taps that fall on it read only zero
    padding.  The output must match PyTorch's shape and the float64 convolution bit for bit."""
    results = [run_lattice(2, H, W, Cin, 24, KH, KW, 2, pad, 9000 + Cin + H + W, res=True, gamma=True) for Cin in (8, 72)]
    report_bitwise(results, f"{KH}x{KW}/s2/p{pad} on {H}x{W}")


# ---------------------------------------------------------------------------------------------------------------- GroupNorm
GN_GS = (1, 2, 3, 4, 6, 8, 12, 24, 64, 256)


def gn_cout(gs, auto):
    if gs == 256:
        return 512
    if gs == 64:
        return 320
    return 256 if auto and gs <= 2 else 264


def gn_cases():
    for gs in GN_GS:
        yield pytest.param(gs, 0, id=f"gs{gs}-auto")
        for bn in BLOCK_NS:
            if (bn % 1000) % gs == 0 and (bn % 1000) // gs <= 64:
                yield pytest.param(gs, bn, id=f"gs{gs}-bn{bn}")


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def gn_run(B, H, W, Cin, Cout, gs, KH, stride, pad, block_n, seed):
    """GroupNorm statistics on exact operands, added onto a pre-filled buffer: each w row has two +-1 entries and x lies in
    [-3, 3], so |acc| <= 6; the bias is a multiple of 1/8 with |bias| <= 2.  The output is checked bit for bit as well."""
    g = G(seed)
    G_ = Cout // gs
    x = lattice((B, H, W, Cin), g).to(dev).bfloat16()
    w = torch.zeros(Cout, Cin * KH * KH, dtype=torch.float64)
    for k in range(2):
        w[torch.arange(Cout), torch.randint(0, Cin * KH * KH, (Cout,), generator=g)] += torch.randint(0, 2, (Cout,), generator=g) * 2 - 1
    w = w.reshape(Cout, Cin, KH, KH)
    wp = ops.pack_conv_weight(w.float().to(dev))
    b = (torch.randint(-16, 17, (Cout,), generator=g).double() / 8).float().to(dev)
    pre = conv64(x, w.to(dev), stride, pad) + b.double()
    assert pre.abs().max().item() <= 8, "exactness premise: |pre| <= 8"
    fill = torch.randint(-2 ** 40, 2 ** 40, (B + 1, G_, 2), generator=g, dtype=torch.int64).to(dev)  # + a guard image
    stbuf = fill.clone()
    out = ops.conv2d(x, wp, KH, KH, stride, pad, bias=b, gn_stats=stbuf[:B], gn_groups=G_, block_n=block_n)
    tag = f"gn_stats B={B} {H}x{W} Cin={Cin} Cout={Cout} gs={gs} {KH}x{KH}/s{stride} bn={block_n}"
    assert torch.equal(stbuf[B], fill[B]), f"{tag}: guard image after the statistics changed"
    st, fill = stbuf[:B], fill[:B]
    pg = pre.reshape(B, -1, G_, gs)
    want = fill + (torch.stack([pg.sum((1, 3)), (pg * pg).sum((1, 3))], -1) * FIX).long()
    if not torch.equal(st, want):
        bad = (st != want).nonzero()
        i = tuple(bad[0].tolist())
        raise AssertionError(f"{tag}: {bad.shape[0]} of {st.numel()} statistics differ, first (image, group, moment) {i}: "
                             f"got {(st - fill)[i].item() / FIX} want {(want - fill)[i].item() / FIX}")
    assert torch.equal(out, emulate(pre - b.double(), b)), f"{tag}: output differs from the emulated epilogue"
    print(f"exact: {st.numel()} statistics and {out.numel()} outputs  {tag}")
    return pre


@pytest.mark.parametrize("gs,block_n", list(gn_cases()))
def test_gn_stats_exact(gs, block_n):
    """Every group size at every N tile that takes it (and the heuristic's pick): 3 images of 75 x 120 pixels as a flat conv, 71
    M tiles per image with a partial last one, 213 in all (odd: the cluster variant runs a padding tile, which addresses image 3,
    the guard image after the statistics), and at least three tiles per persistent CTA (so both parity slot arrays are reused)."""
    Cout = gn_cout(gs, block_n == 0)
    bn = block_n % 1000
    if bn:
        clu = 2 if block_n > 1000 else 1
        items = -(-Cout // bn) * -(-213 // clu)
        grid = min(items * clu, sms()) // clu * clu
        assert items * clu / grid >= 3, "multi-pass premise"
    pre = gn_run(3, 75, 120, 24, Cout, gs, 1, 1, 0, block_n, 31 * gs + block_n)
    assert pre.abs().max().item() >= 4  # the sums are not dominated by zeros


@pytest.mark.parametrize("block_n", [0, 64, 1192])
def test_gn_stats_exact_stride2(block_n):
    """The PAFPN bu_conv2 shape: 3x3 / s2 / p1 with GroupNorm (group size 8), on 2 images of odd size."""
    gn_run(2, 41, 57, 64, 264 if block_n != 1192 else 192, 8, 3, 2, 1, block_n, 5 + block_n)


@pytest.mark.parametrize("block_n,gs", [(128, 1), (256, 2), (1256, 2), (96, 1)])
def test_gn_tile_with_too_many_groups_is_rejected(block_n, gs):
    """An N tile holding more than 64 GroupNorm groups would overflow the CTA's accumulator slots: rejected before launch."""
    x = torch.zeros(1, 4, 4, 8, dtype=torch.bfloat16, device=dev)
    wp = torch.zeros(256, 1, 8, dtype=torch.bfloat16, device=dev)
    st = torch.zeros(1, 256 // gs, 2, dtype=torch.int64, device=dev)
    with pytest.raises(UnicornB200Error, match="GroupNorm groups, more than the 64"):
        ops.conv2d(x, wp, 1, 1, gn_stats=st, gn_groups=256 // gs, block_n=block_n)
    assert not st.any()


# ---------------------------------------------------------------------------------------------------------------- production
# (B, H, W, Cin, Cout, K): the ConvNeXt-L pwconvs at C >= 768 (1x1, Cin up to 6144) and the neck / ResNet 3x3 convs
PROD = [(3, 9, 11, 768, 264, 1), (2, 5, 13, 1536, 136, 1), (2, 7, 9, 3072, 200, 1), (1, 11, 12, 6144, 136, 1),
        (3, 10, 14, 256, 200, 3), (2, 9, 7, 512, 264, 3)]
PROD_CONFIGS = ["bias", "bias_f16out", "f32out", "relu", "gelu", "res_gamma", "relu_res", "gn", "any_f16x", "any_silu",
                "any_f16res"]


def prod_run(B, H, W, Cin, Cout, K, name, seed, drop_last_chunk=False, x=None):
    c = CONFIGS[name]
    g = G(seed)
    xdt, odt, act = c.get("x_dtype", torch.bfloat16), c.get("out_dtype", torch.bfloat16), c.get("act", "none")
    x0 = torch.randn(B, H, W, Cin, generator=g).to(dev).to(xdt)
    x = x0 if x is None else x
    wp = ops.pack_conv_weight((torch.randn(Cout, Cin, K, K, generator=g) / math.sqrt(Cin * K * K)).to(dev), xdt)
    b = torch.randn(Cout, generator=g).to(dev)
    gm = (0.5 * torch.randn(Cout, generator=g)).to(dev) if c.get("gamma") else None
    has_res = c.get("res") or c.get("act_after_res")
    r = torch.randn(x.shape[0], H, W, Cout, generator=g).to(dev).to(odt) if has_res else None
    kw = dict(bias=b, act=ACTS[act], gamma=gm, res=r, act_after_res=c.get("act_after_res", False), out_dtype=odt)
    if c.get("gn"):
        kw.update(gn_stats=torch.zeros(x.shape[0], Cout // 8, 2, dtype=torch.int64, device=dev), gn_groups=Cout // 8)
    out = ops.conv2d(x, wp, K, K, 1, K // 2, **kw)
    w = unpack(wp, Cout, K, K)
    wr = w.clone()
    if drop_last_chunk:
        wr[:, (Cin - 1) // 64 * 64:, K - 1, K - 1] = 0
    pre = conv64(x, wr, 1, K // 2) + b.double()
    S = conv64(x.abs(), w.abs(), 1, K // 2) + b.double().abs()
    if c.get("act_after_res"):
        ref = torch.relu(pre + r.double())
    else:
        ref = act64(pre, act)
    gmd = gm.double() if gm is not None else torch.ones(Cout, dtype=torch.float64, device=dev)
    if not c.get("act_after_res"):
        ref = ref * gmd
        if r is not None:
            ref = ref + r.double()
    lip = ACT_LIP if act in ("gelu", "silu", "sigmoid") else 1.0
    bound = REL[odt] * ref.abs() + gmd.abs() * lip * Cin * K * K * U * S + 2.0 ** -22 * (
        (r.double().abs() if r is not None else 0) + gmd.abs() * pre.abs()) + 1e-6
    if act in ("gelu", "silu", "sigmoid"):
        bound = bound + gmd.abs() * (GELU_FIT + ulp(ref, odt))
    return x, out, ref, bound


@pytest.mark.parametrize("shape", PROD, ids=[f"{K}x{K}-Cin{Cin}" for *_, Cin, _, K in PROD])
def test_production_magnitudes_per_element(shape):
    """Gaussian operands at the real K, every epilogue variant, per element against float64; a reference without the last
    64-channel chunk of the last tap fails the same check; a B > 1 launch gives each image the bits of its B = 1 launch."""
    B, H, W, Cin, Cout, K = shape
    i = PROD.index(shape)
    for j, name in enumerate(PROD_CONFIGS):
        if (i + j) % 2 and name not in ("bias", "res_gamma"):
            continue  # each variant on half the shapes; bias and res_gamma on all
        x, out, ref, bound = prod_run(B, H, W, Cin, Cout, K, name, 100 * i + j)
        check(out, ref, bound, f"[{config_variant(name)}] {name} B={B} {H}x{W} Cin={Cin} Cout={Cout} {K}x{K}")
        if name == "res_gamma":
            _, _, ref_d, bound_d = prod_run(B, H, W, Cin, Cout, K, name, 100 * i + j, drop_last_chunk=True)
            with pytest.raises(AssertionError):
                check(out, ref_d, bound_d, f"{name} Cin={Cin} vs reference without the last chunk of the last tap (must fail)")
        if B > 1 and name in ("bias", "gn"):
            for k in range(B):
                _, one, _, _ = prod_run(B, H, W, Cin, Cout, K, name, 100 * i + j, x=x[k:k + 1].contiguous())
                assert torch.equal(out[k], one[0]), f"{name} Cin={Cin}: image {k} differs from its B = 1 launch"

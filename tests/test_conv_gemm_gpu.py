"""uc_conv2d (wgmma implicit GEMM) against torch fp32 conv2d on the same bf16-rounded operands."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

CASES = [
    # name, B,H,W,Cin,Cout,K,stride,pad, extras
    ("linear_small", 1, 1, 256, 64, 64, 1, 1, 0, {}),
    ("linear_k192_n768_gelu", 1, 1, 1000, 192, 768, 1, 1, 0, {"bias": True, "act": "gelu"}),
    ("linear_res_gamma", 1, 1, 777, 768, 192, 1, 1, 0, {"bias": True, "gamma": True, "res": True}),
    ("linear_cin96", 1, 1, 300, 96, 384, 1, 1, 0, {"bias": True}),
    ("conv1x1_map", 1, 25, 40, 1536, 768, 1, 1, 0, {}),
    ("conv3x3", 1, 50, 80, 256, 256, 3, 1, 1, {"bias": True, "act": "relu"}),
    ("conv3x3_odd", 2, 13, 21, 64, 128, 3, 1, 1, {"act": "silu"}),
    ("conv3x3_s2", 1, 50, 80, 384, 384, 3, 2, 1, {}),
    ("conv3x3_s2_odd", 1, 25, 41, 128, 64, 3, 2, 1, {}),
    ("conv2x2_s2", 1, 40, 64, 192, 384, 2, 2, 0, {"bias": True}),
    ("pred16_f32", 1, 20, 20, 256, 16, 1, 1, 0, {"bias": True, "out_f32": True}),
    ("conv3x3_gn", 1, 20, 36, 256, 256, 3, 1, 1, {"gn": 16}),
    ("conv1x1_gn384", 1, 20, 36, 768, 384, 1, 1, 0, {"gn": 16}),
    ("slice_in_out", 1, 16, 24, 128, 192, 1, 1, 0, {"slice": True}),
    ("f16_embed", 1, 20, 32, 256, 128, 3, 1, 1, {"bias": True, "f16": True}),
]
for bn in (16, 32, 64, 96, 128, 192, 256):
    CASES.append((f"bn{bn}", 1, 1, 640, 320, 768, 1, 1, 0, {"block_n": bn}))
# 2-CTA cluster variant with weight multicast (odd number of M tiles -> one padding tile; GN; 3x3; residual)
for bn in (1128, 1192, 1256):
    CASES.append((f"mc{bn}", 1, 1, 1150, 320, 768, 1, 1, 0, {"block_n": bn, "bias": True, "act": "gelu"}))
CASES.append(("mc_conv3x3_gn", 1, 26, 40, 256, 256, 3, 1, 1, {"block_n": 1256, "gn": 16}))
CASES.append(("mc_res_gamma", 1, 1, 777, 768, 192, 1, 1, 0, {"block_n": 1192, "bias": True, "gamma": True, "res": True}))
CASES.append(("mc_conv3x3_s2", 1, 50, 80, 384, 384, 3, 2, 1, {"block_n": 1128}))
# the fp16 operand path of the explicit N tiles, on a partial last M tile
for bn in (128, 192, 256, 1256):
    CASES.append((f"f16_bn{bn}_gelu", 1, 1, 1150, 320, 768, 1, 1, 0, {"block_n": bn, "bias": True, "act": "gelu", "f16": True}))


def _act(x, name):
    return {None: lambda t: t, "relu": F.relu, "gelu": F.gelu, "silu": F.silu, "sigmoid": torch.sigmoid}[name](x)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_conv(case):
    from unicorn_b200 import ops
    name, B, H, W, Cin, Cout, K, s, pad, ex = case
    g = torch.Generator(device="cpu").manual_seed(hash(name) % (2 ** 31))
    dt = torch.float16 if ex.get("f16") else torch.bfloat16
    dev = "cuda"
    x = torch.randn(B, H, W, Cin, generator=g).to(dev).to(dt)
    w = (torch.randn(Cout, Cin, K, K, generator=g) / (Cin * K * K) ** 0.5).to(dev)
    wp = ops.pack_conv_weight(w, dt)
    bias = torch.randn(Cout, generator=g).to(dev) if ex.get("bias") else None
    gamma = torch.randn(Cout, generator=g).to(dev) if ex.get("gamma") else None
    Ho = (H + 2 * pad - K) // s + 1
    Wo = (W + 2 * pad - K) // s + 1
    res = torch.randn(B, Ho, Wo, Cout, generator=g).to(dev).to(dt) if ex.get("res") else None
    xin = x
    out = None
    if ex.get("slice"):
        big = torch.zeros(B, H, W, Cin + 64, device=dev, dtype=dt)
        big[..., 32:32 + Cin] = x
        xin = big[..., 32:32 + Cin]
        obig = torch.full((B, Ho, Wo, Cout + 64), 7.0, device=dev, dtype=dt)
        out = obig[..., 8:8 + Cout]
    gn_stats = torch.zeros(B, ex["gn"], 2, device=dev, dtype=torch.int64) if ex.get("gn") else None
    act = ex.get("act")
    y = ops.conv2d(xin, wp, K, K, s, pad, bias=bias, act=getattr(ops, "ACT_" + act.upper()) if act else 0,
                   gamma=gamma, res=res, out=out, out_dtype=torch.float32 if ex.get("out_f32") else None,
                   block_n=ex.get("block_n", 0), gn_stats=gn_stats, gn_groups=ex.get("gn", 0))
    torch.cuda.synchronize()
    # reference on identical (rounded) operands, fp32 math
    xr = x.float().permute(0, 3, 1, 2)
    wr = wp[:Cout].float().reshape(Cout, K, K, Cin).permute(0, 3, 1, 2)
    pre = F.conv2d(xr, wr, bias, stride=s, padding=pad)
    ref = _act(pre, act)
    if gamma is not None:
        ref = ref * gamma.view(1, -1, 1, 1)
    if res is not None:
        ref = ref + res.float().permute(0, 3, 1, 2)
    ref = ref.permute(0, 2, 3, 1)
    got = y.float()
    err = (got - ref).abs().max().item()
    scale = ref.abs().max().item()
    tol = (4e-3 if y.dtype != torch.float32 else 2e-5) * scale + 1e-3
    assert err <= tol, f"{name}: max err {err:.4g} (scale {scale:.3g}, tol {tol:.3g})"
    if ex.get("slice"):
        assert (obig[..., :8] == 7).all() and (obig[..., 8 + Cout:] == 7).all()
    if gn_stats is not None:
        G = ex["gn"]
        pg = pre.reshape(B, G, Cout // G, Ho * Wo)
        s1 = pg.sum(dim=(2, 3))
        s2 = (pg * pg).sum(dim=(2, 3))
        st = gn_stats.double() / 2 ** 22
        assert torch.allclose(st[..., 0].float(), s1, rtol=2e-3, atol=2e-1), (st[..., 0], s1)
        assert torch.allclose(st[..., 1].float(), s2, rtol=2e-3, atol=2e-1), (st[..., 1], s2)


def test_gelu_epilogue_whole_range():
    """The GELU of the epilogue (uc_epilogue.cuh: x * sigmoid(x * P(x^2)) on fp32 pairs) over the whole range a pre-activation can
    take, including values whose exponentials saturate or overflow: a 1x1 conv with the identity as weight and the test values as
    bias.  fp32 output against torch's exact GELU."""
    from unicorn_b200 import ops
    C = 64
    vals = torch.cat([torch.linspace(-12, 12, 4001), torch.tensor([-1e4, -300.0, -88.0, -40.0, -20.0, 0.0, -0.0, 20.0, 88.0, 300.0, 1e4, 3e38, -3e38])])
    n = vals.numel()
    rows = -(-n // C)
    b = torch.zeros(rows * C)
    b[:n] = vals
    x = torch.zeros(1, 1, rows, C, device="cuda", dtype=torch.bfloat16)
    w = ops.pack_conv_weight(torch.eye(C, device="cuda").view(C, C, 1, 1))
    got = torch.cat([ops.conv2d(x[:, :, r:r + 1].contiguous(), w, 1, 1, bias=b[r * C:(r + 1) * C].cuda().contiguous(), act=ops.ACT_GELU,
                                out_dtype=torch.float32).view(-1) for r in range(rows)])[:n].cpu()
    ref = F.gelu(vals.double()).float()
    assert torch.isfinite(got).all()
    err = (got - ref).abs()
    assert (err <= 1e-5 + 1e-5 * ref.abs()).all(), (err.max(), vals[err.argmax()])
    # saturation: exactly zero far on the negative side, the identity far on the positive side
    assert got[vals == -1e4].abs().max() == 0 and abs(got[(vals - 12).abs().argmin()] - 12.0) < 1e-4

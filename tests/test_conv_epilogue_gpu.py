"""uc_conv2d's epilogue variants (one kernel instantiation per feature set, conv_gemm.cuh) against torch fp32 on the same rounded
operands, at every N tile with partial M and N tiles; and the fixed variants bit-identical to the run-time-tested one (kEpiAny)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

BLOCK_NS = (16, 96, 128, 192, 256, 1128, 1256)

# name: conv2d keywords (see _run); "gn" = (groups, Cout)
VARIANTS = {
    "bias": dict(bias=True),
    "bias_f16out": dict(bias=True, out=torch.float16),
    "f32out": dict(bias=True, out=torch.float32),
    "no_bias": dict(),
    "relu": dict(bias=True, act="relu"),
    "gelu": dict(bias=True, act="gelu"),
    "gelu_ln": dict(bias=True, act="gelu", ln=True),
    "res_gamma": dict(bias=True, gamma=True, res=True),
    "res": dict(bias=True, res=True),
    "relu_res": dict(bias=True, act="relu", res=True, act_after_res=True),
    "gn4": dict(bias=True, gn=(50, 200)),
    "gn24": dict(bias=True, gn=(8, 192)),
    # kEpiAny: combinations the fixed variants do not cover
    "silu": dict(bias=True, act="silu"),
    "sigmoid": dict(bias=True, act="sigmoid"),
    "gelu_gamma": dict(bias=True, act="gelu", gamma=True),
    "relu_gn4": dict(bias=True, act="relu", gn=(50, 200)),
    "f16x_gelu_res": dict(bias=True, act="gelu", gamma=True, res=True, x=torch.float16),
    "f16x_gn4": dict(bias=True, gn=(50, 200), x=torch.float16),
}


def _cases():
    for name, v in VARIANTS.items():
        for bn in BLOCK_NS:
            gs = v["gn"][1] // v["gn"][0] if "gn" in v else 0
            if gs and (bn % 1000) % gs:
                continue
            yield pytest.param(name, bn, "linear", id=f"{name}-{bn}-linear")
            if bn in (16, 128, 256, 1256) and "ln" not in v:  # the folded LayerNorm is for 1x1 convs only
                yield pytest.param(name, bn, "3x3", id=f"{name}-{bn}-3x3")
    for bn in (96, 192, 1192):
        yield pytest.param("gn24", bn, "3x3", id=f"gn24-{bn}-3x3")


def _operands(name, shape, seed):
    from unicorn_b200 import ops
    v = VARIANTS[name]
    dt = v.get("x", torch.bfloat16)
    Cout = v["gn"][1] if "gn" in v else 200
    # linear: M = 1150 = 8 full 128-pixel tiles + a partial one (odd tile count: a padding tile in the cluster variant);
    # 3x3: 2 images of 13 x 21, partial 2-D tiles.  Cout 200 / 192: the last N tile is partial for most block_n.
    B, H, W, Cin, K, pad = (1, 1, 1150, 192, 1, 0) if shape == "linear" else (2, 13, 21, 64, 3, 1)
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(B, H, W, Cin, generator=g).cuda().to(dt)
    w = (torch.randn(Cout, Cin, K, K, generator=g) / (Cin * K * K) ** 0.5).cuda()
    wp = ops.pack_conv_weight(w, dt)
    bias = torch.randn(Cout, generator=g).cuda() if v.get("bias") else None
    gamma = torch.randn(Cout, generator=g).cuda() if v.get("gamma") else None
    ydt = v.get("out", dt)
    res = torch.randn(B, H, W, Cout, generator=g).cuda().to(ydt) if v.get("res") else None
    return dict(x=x, wp=wp, K=K, pad=pad, bias=bias, gamma=gamma, res=res, ydt=ydt)


def _ln_fold(x, wp):
    """row_stats / col_s of a LayerNorm folded into the 1x1 conv (eps 1e-6), and the reference's per-pixel (mu, rstd)."""
    xd = x.reshape(-1, x.shape[3]).double()
    rs = torch.stack([(xd.sum(1) * 2 ** 22).round(), ((xd * xd).sum(1) * 2 ** 22).round()], 1).to(torch.int64).contiguous()
    col_s = wp.float().reshape(wp.shape[0], -1).sum(1).contiguous()
    mu = xd.mean(1)
    rstd = 1.0 / torch.sqrt(xd.var(1, unbiased=False) + 1e-6)
    return rs, col_s, mu.float(), rstd.float()


def _run(name, o, bn, **over):
    from unicorn_b200 import ops
    v = VARIANTS[name]
    act = v.get("act")
    kw = dict(bias=o["bias"], act=getattr(ops, "ACT_" + act.upper()) if act else 0, gamma=o["gamma"], res=o["res"],
              out_dtype=o["ydt"], block_n=bn, act_after_res=v.get("act_after_res", False))
    st = None
    if "gn" in v:
        st = torch.zeros(o["x"].shape[0], v["gn"][0], 2, device="cuda", dtype=torch.int64)
        kw.update(gn_stats=st, gn_groups=v["gn"][0])
    if v.get("ln"):
        rs, col_s, _, _ = _ln_fold(o["x"], o["wp"])
        kw.update(row_stats=rs, col_s=col_s, row_eps=1e-6)
    kw.update(over)
    y = ops.conv2d(o["x"], o["wp"], o["K"], o["K"], 1, o["pad"], **kw)
    return y, st


def _act(t, name):
    return {None: lambda a: a, "relu": F.relu, "gelu": F.gelu, "silu": F.silu, "sigmoid": torch.sigmoid}[name](t)


@pytest.mark.parametrize("name,block_n,shape", list(_cases()))
def test_epilogue_variant(name, block_n, shape):
    v = VARIANTS[name]
    o = _operands(name, shape, block_n * 7 + len(name))
    y, st = _run(name, o, block_n)
    torch.cuda.synchronize()
    x, wp, K, pad = o["x"], o["wp"], o["K"], o["pad"]
    Cout, Cin = wp.shape[0], x.shape[3]
    wr = wp.float().reshape(Cout, K, K, Cin).permute(0, 3, 1, 2)
    pre = F.conv2d(x.float().permute(0, 3, 1, 2), wr, None, padding=pad)
    if v.get("ln"):
        _, col_s, mu, rstd = _ln_fold(x, wp)
        B, _, H, W = pre.shape
        r = rstd.view(B, H, W, 1).permute(0, 3, 1, 2)
        pre = r * pre - (r * mu.view(B, H, W, 1).permute(0, 3, 1, 2)) * col_s.view(1, -1, 1, 1)
    if o["bias"] is not None:
        pre = pre + o["bias"].view(1, -1, 1, 1)
    res = o["res"].float().permute(0, 3, 1, 2) if o["res"] is not None else None
    if v.get("act_after_res"):
        ref = F.relu(pre + res)
    else:
        ref = _act(pre, v.get("act"))
        if o["gamma"] is not None:
            ref = ref * o["gamma"].view(1, -1, 1, 1)
        if res is not None:
            ref = ref + res
    ref = ref.permute(0, 2, 3, 1)
    assert y.dtype == o["ydt"]
    err = (y.float() - ref).abs().max().item()
    tol = (1e-4 if y.dtype == torch.float32 else 4e-3) * ref.abs().max().item() + 1e-3
    assert err <= tol, f"max err {err:.4g} (tol {tol:.3g})"
    if st is not None:
        G = v["gn"][0]
        pg = pre.reshape(pre.shape[0], G, Cout // G, -1)
        got = st.double() / 2 ** 22
        assert torch.allclose(got[..., 0].float(), pg.sum(dim=(2, 3)), rtol=2e-3, atol=2e-1)
        assert torch.allclose(got[..., 1].float(), (pg * pg).sum(dim=(2, 3)), rtol=2e-3, atol=2e-1)


# a fixed variant, and an extra argument that changes nothing numerically but sends the same call to kEpiAny
SAME_AS_ANY = {
    "bias": dict(gamma="ones"),
    "relu": dict(gamma="ones"),
    "gelu": dict(gamma="ones"),
    "f32out": dict(gamma="ones"),
    "gn4": dict(gamma="ones"),
    "gn24": dict(gamma="ones"),
    "res": dict(gn=True),
}


@pytest.mark.parametrize("name", list(SAME_AS_ANY))
@pytest.mark.parametrize("block_n", (16, 96, 192, 256, 1192))
def test_fixed_variant_matches_any(name, block_n):
    """x * 1.0 is exact, and GroupNorm statistics do not change the output: the fixed variant and kEpiAny give the same bits, for the
    output and for the statistics."""
    v = VARIANTS[name]
    gs = v["gn"][1] // v["gn"][0] if "gn" in v else 0
    if gs and (block_n % 1000) % gs:
        pytest.skip("N tile incompatible with the group size")
    o = _operands(name, "3x3", block_n + 11)
    y, st = _run(name, o, block_n)
    Cout = o["wp"].shape[0]
    over = {}
    if SAME_AS_ANY[name].get("gamma"):
        over["gamma"] = torch.ones(Cout, device="cuda")
    st2 = None
    if SAME_AS_ANY[name].get("gn"):
        st2 = torch.zeros(o["x"].shape[0], 25, 2, device="cuda", dtype=torch.int64)
        over.update(gn_stats=st2, gn_groups=25)
    y2, st3 = _run(name, o, block_n, **over)
    torch.cuda.synchronize()
    assert torch.equal(y.view(torch.uint8), y2.view(torch.uint8))
    if st is not None:
        assert torch.equal(st, st3)

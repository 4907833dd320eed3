"""uc_conv2d's 16-bit epilogue, which loads the residual and stores the output tile by TMA through a shared-memory staging tile:
channel-slice outputs whose width is not a multiple of the staging slab, partial 2-D tiles, staging reuse across many tiles per CTA,
and in-place residuals (res is y)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

BLOCK_NS = (16, 32, 64, 96, 128, 192, 256, 1128, 1192, 1256)


def _operands(seed, B, H, W, Cin, Cout, K, s, pad, dt=torch.bfloat16):
    from unicorn_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(B, H, W, Cin, generator=g).cuda().to(dt)
    w = (torch.randn(Cout, Cin, K, K, generator=g) / (Cin * K * K) ** 0.5).cuda()
    wp = ops.pack_conv_weight(w, dt)
    Ho, Wo = (H + 2 * pad - K) // s + 1, (W + 2 * pad - K) // s + 1
    bias = torch.randn(Cout, generator=g).cuda()
    gamma = torch.randn(Cout, generator=g).cuda()
    res = torch.randn(B, Ho, Wo, Cout, generator=g).cuda().to(dt)
    return x, wp, bias, gamma, res


def _reference(x, wp, K, s, pad, bias, act=None, gamma=None, res=None, act_after_res=False):
    Cout, Cin = wp.shape[0], x.shape[3]
    wr = wp.float().reshape(Cout, K, K, Cin).permute(0, 3, 1, 2)
    pre = F.conv2d(x.float().permute(0, 3, 1, 2), wr, bias, stride=s, padding=pad)
    if act_after_res:
        return F.relu(pre + res.float().permute(0, 3, 1, 2)).permute(0, 2, 3, 1), pre
    y = {None: lambda t: t, "relu": F.relu, "gelu": F.gelu}[act](pre)
    if gamma is not None:
        y = y * gamma.view(1, -1, 1, 1)
    if res is not None:
        y = y + res.float().permute(0, 3, 1, 2)
    return y.permute(0, 2, 3, 1), pre


def _check(got, ref, what):
    err = (got.float() - ref).abs().max().item()
    tol = 4e-3 * ref.abs().max().item() + 1e-3
    assert err <= tol, f"{what}: max err {err:.4g} (tol {tol:.3g})"


@pytest.mark.parametrize("block_n", BLOCK_NS)
def test_residual_gamma_slice(block_n):
    """Cout 136 is not a multiple of any slab of 32 or 64 columns: the last slab is clipped at Cout by the store, and the guard columns
    on both sides of the output slice keep their 7.0.  The residual is a channel slice of another buffer."""
    from unicorn_b200 import ops
    Cout = 136
    x, wp, bias, gamma, res = _operands(block_n, 1, 1, 1150, 192, Cout, 1, 1, 0)
    rbig = torch.full((1, 1, 1150, Cout + 24), -5.0, device="cuda", dtype=torch.bfloat16)
    rbig[..., 16:16 + Cout] = res
    obig = torch.full((1, 1, 1150, Cout + 64), 7.0, device="cuda", dtype=torch.bfloat16)
    out = obig[..., 8:8 + Cout]
    ops.conv2d(x, wp, 1, 1, bias=bias, act=ops.ACT_GELU, gamma=gamma, res=rbig[..., 16:16 + Cout], out=out, block_n=block_n)
    torch.cuda.synchronize()
    ref, _ = _reference(x, wp, 1, 1, 0, bias, "gelu", gamma, res)
    _check(out, ref, f"block_n {block_n}")
    assert (obig[..., :8] == 7).all() and (obig[..., 8 + Cout:] == 7).all()


@pytest.mark.parametrize("shape", [(2, 13, 21, 1, 128), (1, 25, 41, 2, 256)], ids=["13x21", "25x41_s2"])
@pytest.mark.parametrize("gn", [False, True], ids=["res", "gn"])
def test_partial_2d_tiles(shape, gn):
    """3x3 convs whose 2-D pixel tiles are partial in both dimensions: the residual box is zero-filled and the store clipped there."""
    from unicorn_b200 import ops
    B, H, W, s, Cout = shape
    x, wp, bias, gamma, res = _operands(H * W + gn, B, H, W, 128, Cout, 3, s, 1)
    G = 16
    st = torch.zeros(B, G, 2, device="cuda", dtype=torch.int64) if gn else None
    y = ops.conv2d(x, wp, 3, 3, s, 1, bias=bias, act=ops.ACT_RELU, gamma=None if gn else gamma, res=None if gn else res,
                   gn_stats=st, gn_groups=G if gn else 0)
    torch.cuda.synchronize()
    ref, pre = _reference(x, wp, 3, s, 1, bias, "relu", None if gn else gamma, None if gn else res)
    _check(y, ref, f"{shape} gn={gn}")
    if gn:
        pg = pre.reshape(B, G, Cout // G, -1)
        got = st.double() / 2 ** 22
        assert torch.allclose(got[..., 0].float(), pg.sum(dim=(2, 3)), rtol=2e-3, atol=2e-1)
        assert torch.allclose(got[..., 1].float(), (pg * pg).sum(dim=(2, 3)), rtol=2e-3, atol=2e-1)


@pytest.mark.parametrize("block_n", [64, 128, 256, 1256])
def test_staging_reuse_many_tiles(block_n):
    """M = 20000 x 256 -> 768: every CTA runs at least 4 tiles through the one staging tile."""
    from unicorn_b200 import ops
    x, wp, bias, gamma, res = _operands(7, 1, 1, 20000, 256, 768, 1, 1, 0)
    y = ops.conv2d(x, wp, 1, 1, bias=bias, act=ops.ACT_GELU, gamma=gamma, res=res, block_n=block_n)
    torch.cuda.synchronize()
    ref, _ = _reference(x, wp, 1, 1, 0, bias, "gelu", gamma, res)
    _check(y, ref, f"block_n {block_n}")


@pytest.mark.parametrize("block_n", BLOCK_NS)
@pytest.mark.parametrize("act_after_res", [False, True], ids=["res_gamma", "act_after_res"])
def test_in_place_residual_bit_identical(block_n, act_after_res):
    """res is y: the result is bit-identical to the same call out of place, and a second identical launch repeats it bit for bit."""
    from unicorn_b200 import ops
    x, wp, bias, gamma, res = _operands(block_n + act_after_res, 2, 19, 37, 192, 200, 3, 1, 1)
    kw = dict(bias=bias, act=ops.ACT_RELU, block_n=block_n, act_after_res=act_after_res, gamma=None if act_after_res else gamma)
    y_out = ops.conv2d(x, wp, 3, 3, 1, 1, res=res, **kw)
    y_in = res.clone()
    ops.conv2d(x, wp, 3, 3, 1, 1, res=y_in, out=y_in, **kw)
    y_again = ops.conv2d(x, wp, 3, 3, 1, 1, res=res, **kw)
    torch.cuda.synchronize()
    ref, _ = _reference(x, wp, 3, 1, 1, bias, "relu", kw["gamma"], res, act_after_res)
    _check(y_out, ref, f"block_n {block_n}")
    assert torch.equal(y_in.view(torch.int16), y_out.view(torch.int16))
    assert torch.equal(y_again.view(torch.int16), y_out.view(torch.int16))

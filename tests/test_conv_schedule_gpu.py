"""uc_conv2d across the persistent schedule of conv_gemm.cuh: shapes that give a CTA 1, 2, 3 or 5 work items, one-step K loops,
partial M tiles and Cout edges, an in-place residual, GroupNorm statistics, fp32 output and the 2-CTA cluster variant.  Each is
checked against torch fp32, bit for bit across every N tile the layer accepts (an output element's K order does not depend on the
N tile, so the per-layer N-tile tables cannot change results), and bit for bit across two launches."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

BLOCK_NS = (16, 32, 64, 96, 128, 192, 256, 1128, 1192, 1256)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# name: (items per CTA at N tile 128 with one N tile, Cin, K, Cout, features).  M = items * SMs * 128 - 40: the last M tile is
# partial, and Cout 120 / 200 leave a partial last N tile for most N tiles.
CASES = {
    "one_item_k1_gelu": (1, 64, 1, 120, dict(act="gelu")),
    "two_items_k1_gelu": (2, 64, 1, 120, dict(act="gelu")),
    "three_items_k2_res_inplace": (3, 128, 1, 120, dict(gamma=True, res="inplace")),
    "three_items_k5_res": (3, 320, 1, 200, dict(gamma=True, res=True)),
    "two_items_k9_3x3_gn": (2, 64, 3, 200, dict(gn=50)),
    "three_items_k1_gn": (3, 64, 1, 120, dict(gn=30)),
    "two_items_k3_f32": (2, 192, 1, 120, dict(out=torch.float32)),
    "five_items_k12_gelu": (5, 768, 1, 128, dict(act="gelu")),
}


def _accepts(bn, ex, Cout):
    if "gn" not in ex:
        return True
    return (bn % 1000) % (Cout // ex["gn"]) == 0


def _operands(name):
    from unicorn_b200 import ops
    ipc, Cin, K, Cout, ex = CASES[name]
    M = ipc * _sms() * 128 - 40
    # 3x3: an NHWC map of 16-row strips (partial 2-D tiles); 1x1: one row of M pixels
    B, H, W = (1, 16, M // 16) if K == 3 else (1, 1, M)
    g = torch.Generator(device="cpu").manual_seed(len(name) * 131 + Cin)
    x = torch.randn(B, H, W, Cin, generator=g).cuda().bfloat16()
    w = (torch.randn(Cout, Cin, K, K, generator=g) / (Cin * K * K) ** 0.5).cuda()
    wp = ops.pack_conv_weight(w)
    bias = torch.randn(Cout, generator=g).cuda()
    gamma = torch.randn(Cout, generator=g).cuda() if ex.get("gamma") else None
    ydt = ex.get("out", torch.bfloat16)
    res = torch.randn(B, H, W, Cout, generator=g).cuda().to(ydt) if ex.get("res") else None
    return dict(x=x, wp=wp, K=K, pad=(K - 1) // 2, bias=bias, gamma=gamma, res=res, ydt=ydt, ex=ex, Cout=Cout)


def _run(o, bn):
    from unicorn_b200 import ops
    ex = o["ex"]
    x = o["x"]
    B, H, W, _ = x.shape
    out = torch.empty(B, H, W, o["Cout"], device="cuda", dtype=o["ydt"])
    res = o["res"]
    if ex.get("res") == "inplace":  # res == y: each tile's residual is read before the same tile is stored
        out.copy_(res)
        res = out
    st = None
    kw = {}
    if "gn" in ex:
        st = torch.zeros(B, ex["gn"], 2, device="cuda", dtype=torch.int64)
        kw.update(gn_stats=st, gn_groups=ex["gn"])
    ops.conv2d(x, o["wp"], o["K"], o["K"], 1, o["pad"], bias=o["bias"], act=ops.ACT_GELU if ex.get("act") == "gelu" else 0,
               gamma=o["gamma"], res=res, out=out, block_n=bn, **kw)
    return out, st


@pytest.mark.parametrize("name", list(CASES))
def test_conv_schedule(name):
    o = _operands(name)
    ex, Cout = o["ex"], o["Cout"]
    x, wp, K = o["x"], o["wp"], o["K"]
    Cin = x.shape[3]
    wr = wp[:Cout].float().reshape(Cout, K, K, Cin).permute(0, 3, 1, 2)
    pre = F.conv2d(x.float().permute(0, 3, 1, 2), wr, o["bias"], padding=o["pad"])
    ref = F.gelu(pre) if ex.get("act") == "gelu" else pre
    if o["gamma"] is not None:
        ref = ref * o["gamma"].view(1, -1, 1, 1)
    if o["res"] is not None:
        ref = ref + o["res"].float().permute(0, 3, 1, 2)
    ref = ref.permute(0, 2, 3, 1)
    first = None
    for bn in BLOCK_NS:
        if not _accepts(bn, ex, Cout):
            continue
        y, st = _run(o, bn)
        y2, st2 = _run(o, bn)
        torch.cuda.synchronize()
        err = (y.float() - ref).abs().max().item()
        tol = (1e-4 if y.dtype == torch.float32 else 4e-3) * ref.abs().max().item() + 1e-3
        assert err <= tol, f"block_n {bn}: max err {err:.4g} (tol {tol:.3g})"
        assert torch.equal(y.view(torch.uint8), y2.view(torch.uint8)), f"block_n {bn}: two launches differ"
        if st is not None:
            assert torch.equal(st, st2), f"block_n {bn}: GroupNorm statistics differ between launches"
            G = ex["gn"]
            pg = pre.reshape(pre.shape[0], G, Cout // G, -1)
            got = st.double() / 2 ** 22
            assert torch.allclose(got[..., 0].float(), pg.sum(dim=(2, 3)), rtol=2e-3, atol=2e-1)
            assert torch.allclose(got[..., 1].float(), (pg * pg).sum(dim=(2, 3)), rtol=2e-3, atol=2e-1)
        if first is None:
            first = (bn, y, st)
        else:
            assert torch.equal(y.view(torch.uint8), first[1].view(torch.uint8)), f"block_n {bn} and {first[0]} differ"
            if st is not None:
                assert torch.equal(st, first[2]), f"GroupNorm statistics of block_n {bn} and {first[0]} differ"

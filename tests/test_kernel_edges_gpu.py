"""Edge-case parity of the GroupNorm-apply, LayerNorm, correlation and small data-movement kernels against float64 references on
the same rounded operands: every instantiation their entry points dispatch to, channel slices of wider buffers (whose guard columns
must keep their values), partial blocks, and the inputs where one-pass statistics and online softmax go wrong (constant groups and
rows, a large common offset, near one-hot softmax with the maximum arriving last).

Bounds are per element: |got - ref| <= |ref| * 2^-8 (one bf16 rounding of a 16-bit output; 2^-11 for fp16) + a small absolute floor;
the fp32 output of the correlation has a tighter relative term.  Every check prints its largest err / bound."""
import math

import pytest
import torch
import torch.nn.functional as F

from unicorn_b200 import ops
from unicorn_b200._lib import UnicornB200Error

pytestmark = pytest.mark.gpu
dev = "cuda"
REL = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
FIX = 2.0 ** 22  # fixed-point scale of the GroupNorm statistics (kGnFixedScale)


def G(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def check(got, ref, rel, floor, name):
    """Per-element bound |got - ref| <= |ref| * rel + floor; ref is float64."""
    err = (got.double() - ref).abs()
    ratio = (err / (ref.abs() * rel + floor)).max().item()
    print(f"err/bound {ratio:.3f}  {name}")
    assert ratio <= 1.0, f"{name}: max err/bound {ratio:.3g} (max err {err.max().item():.3g})"
    return ratio


def guarded(lead, C, lo, hi, dtype, seed):
    """A [*lead, lo + C + hi] buffer of random guard values and its channel slice [..., lo:lo + C]."""
    buf = torch.randn(*lead, lo + C + hi, generator=G(seed)).to(dev, dtype)
    return buf, buf[..., lo:lo + C]


def guards_kept(buf, before, lo, C, name):
    assert torch.equal(buf[..., :lo], before[..., :lo]), f"{name}: left guard columns overwritten"
    assert torch.equal(buf[..., lo + C:], before[..., lo + C:]), f"{name}: right guard columns overwritten"


def offset_values(n, base, ratio, dtype, g):
    """n values of the 16-bit dtype with mean ~base and std ~|base| / ratio, all exactly representable: base + k * ulp(base).  When
    the std is below one ulp, a fraction of the values sits one ulp off base (the std is then ulp * sqrt(fraction))."""
    ulp = 2.0 ** (math.floor(math.log2(abs(base))) - (7 if dtype == torch.bfloat16 else 10))
    sigma = abs(base) / ratio
    if sigma >= ulp:
        k = torch.round(torch.randn(n, generator=g, dtype=torch.float64) * sigma / ulp)
    else:
        p = (sigma / ulp) ** 2
        u = torch.rand(n, generator=g, dtype=torch.float64)
        k = (u < p / 2).double() - ((u >= p / 2) & (u < p)).double()
    return base + k * ulp


# ---------------------------------------------------------------------------------------------------------------- GroupNorm apply
ACT_REF = {ops.ACT_NONE: lambda f: f, ops.ACT_RELU: lambda f: f.clamp_min(0), ops.ACT_SILU: F.silu}
GN_FLOOR = 1e-3


def fixed_point_stats(x, G_):
    """{sum, sum of squares} per (image, group) of the stored map in float64, quantised to the 2^22 fixed point of uc_conv2d."""
    B, H, W, C = x.shape
    xd = x.double().reshape(B, H * W, G_, C // G_)
    st = torch.stack([xd.sum((1, 3)), (xd * xd).sum((1, 3))], -1) * FIX
    return st.round().to(torch.int64).contiguous()


def moments(st, n):
    s, q = st[..., 0].double() / FIX, st[..., 1].double() / FIX
    mean = s / n
    return mean, (q / n - mean * mean).clamp_min(0)


def gn_ref(x, mean, var, eps, w, b, act, prior=None, beta=None):
    """act((x - mean) / sqrt(var + eps) * w + b) (+ prior * beta) in float64; x [B,H,W,C], mean / var [B,G]."""
    gs = x.shape[3] // mean.shape[1]
    m = mean.repeat_interleave(gs, 1)[:, None, None, :]
    r = (var + eps).rsqrt().repeat_interleave(gs, 1)[:, None, None, :]
    f = ACT_REF[act]((x.double() - m) * r * w.double() + b.double())
    if prior is not None:
        f = f + prior.double()[..., None] * beta.double()
    return f


def run_gn(x, st, gw, gb, G_, eps, act, inplace, with_prior, with_out2, seed, name):
    """One uc_groupnorm_apply call on channel slices (x, y, add2, y2 8 channels into wider buffers) with the float64 reference of the
    same statistics; returns the largest err / bound."""
    B, H, W, C = x.shape
    g = G(seed)
    xb, xs = guarded((B, H, W), C, 8, 16, torch.bfloat16, seed + 1)
    xs.copy_(x)
    if inplace:
        yb, ys = xb, xs
    else:
        yb, ys = guarded((B, H, W), C, 8, 8, torch.bfloat16, seed + 2)
    prior = beta = add2 = out2 = None
    if with_prior:
        prior = torch.rand(B, H, W, generator=g).to(dev)
        beta = torch.randn(C, generator=g).to(dev)
    if with_out2:
        ab, add2 = guarded((B, H, W), C, 16, 8, torch.bfloat16, seed + 3)
        ob, out2 = guarded((B, H, W), C, 8, 24, torch.bfloat16, seed + 4)
        ob0 = ob.clone()
    xb0, yb0 = xb.clone(), yb.clone()
    mean, var = moments(st, H * W * (C // G_))
    ref = gn_ref(x, mean, var, eps, gw, gb, act, prior, beta)
    ops.groupnorm_apply(xs, st, gw, gb, G_, eps, act, out=None if inplace else ys, prior=prior, beta=beta, add2=add2, out2=out2)
    r = check(ys, ref, REL[torch.bfloat16], GN_FLOOR, name)
    guards_kept(yb, yb0, 8, C, name)
    if not inplace:
        assert torch.equal(xb, xb0), f"{name}: out-of-place call changed its input"
    if with_out2:
        r = max(r, check(out2, ref + add2.double(), REL[torch.bfloat16], GN_FLOOR, name + " out2"))
        guards_kept(ob, ob0, 8, C, name + " out2")
    return r


GN_SHAPES = [  # C, G, (H, W), B
    (8, 1, (1, 1), 1), (8, 1, (1, 37), 3), (256, 1, (1, 37), 1), (256, 16, (1, 37), 3), (256, 32, (1, 1), 3),
    (4096, 1, (1, 37), 1), (4096, 16, (1, 37), 3), (4096, 512, (1, 1), 3),
    # grid-stride loop: 3 x 32000 pixels x 32 8-channel chunks, gx capped at 8 * SMs -> every thread runs several rounds
    (256, 16, (160, 200), 3),
]


@pytest.mark.parametrize("C,G_,HW,B", GN_SHAPES)
def test_groupnorm_apply_shapes(C, G_, HW, B):
    g = G(100 + C + G_)
    x = (torch.randn(B, *HW, C, generator=g) * 1.7 + 0.4).to(dev).bfloat16()
    gw, gb = (1 + 0.3 * torch.randn(C, generator=g)).to(dev), (0.5 * torch.randn(C, generator=g)).to(dev)
    st = fixed_point_stats(x, G_)
    combos = [(False, True, True), (True, False, False), (False, False, True), (True, True, False)]
    if HW[0] * HW[1] > 1000:
        combos = combos[:2]
    for act in ACT_REF:
        for inplace, with_prior, with_out2 in combos:
            run_gn(x, st, gw, gb, G_, 1e-3, act, inplace, with_prior, with_out2, 7,
                   f"gn C={C} G={G_} HW={HW} B={B} act={act} inplace={inplace} prior={with_prior} out2={with_out2}")


def test_groupnorm_apply_constant_groups():
    """Variance 0: rstd = 1/sqrt(eps), the output must be act(b) (+ prior * beta) up to rounding.  Zero and non-zero constants, and
    groups of different constants next to a random group."""
    B, H, W, C, G_ = 2, 6, 7, 64, 8
    g = G(11)
    consts = torch.tensor([0.0, 0.30078125, -3.5, 6.0, 7.25, -0.0078125, 1.5, 0.0]).repeat_interleave(C // G_)
    x = consts.expand(B, H, W, C).clone()
    x[1, ..., 16:24] = torch.randn(H, W, 8, generator=g)  # one ordinary group in image 1
    x = x.to(dev).bfloat16()
    gw, gb = (1 + 0.3 * torch.randn(C, generator=g)).to(dev), torch.randn(C, generator=g).to(dev)
    st = fixed_point_stats(x, G_)
    mean, var = moments(st, H * W * (C // G_))
    assert (var[0] == 0).all() and (var[1, torch.arange(G_, device=dev) != 2] == 0).all()
    for eps in (1e-3, 1e-5):
        for act in ACT_REF:
            run_gn(x, st, gw, gb, G_, eps, act, False, False, True, 12, f"gn constant groups eps={eps} act={act}")
            out = ops.groupnorm_apply(x, st, gw, gb, G_, eps, act, out=torch.empty_like(x))
            want = ACT_REF[act](gb.double()).expand(H, W, C)
            check(out[0], want, REL[torch.bfloat16], GN_FLOOR, f"gn constant groups = act(b), eps={eps} act={act}")


@pytest.mark.parametrize("ratio", [10, 100, 1000])
def test_groupnorm_apply_large_offset(ratio):
    """Groups with |mean| / std = ratio, statistics quantised exactly as uc_conv2d stores them: the apply kernel computes the variance
    in float64 from them and folds it into fp32 scale / shift."""
    B, H, W, C, G_ = 2, 5, 9, 128, 16
    g = G(13)
    n = H * W * (C // G_)
    blocks = [offset_values(n, (768.0 if (b + k) % 2 else -384.0), ratio, torch.bfloat16, g) for b in range(B) for k in range(G_)]
    x = torch.stack(blocks).reshape(B, G_, H * W, C // G_).permute(0, 2, 1, 3).reshape(B, H, W, C).to(dev).bfloat16()
    gw, gb = (1 + 0.3 * torch.randn(C, generator=g)).to(dev), (0.5 * torch.randn(C, generator=g)).to(dev)
    st = fixed_point_stats(x, G_)
    mean, var = moments(st, n)
    print(f"realised |mean|/std: {(mean.abs() / var.sqrt()).min().item():.0f} .. {(mean.abs() / var.sqrt()).max().item():.0f}")
    for act in ACT_REF:
        run_gn(x, st, gw, gb, G_, 1e-3, act, False, True, True, 14, f"gn |mean|/std={ratio} act={act}")


def conv_gn_chain(ratio, G_, eps, seed=15):
    """uc_conv2d with gn_stats, then uc_groupnorm_apply.  The reference applies the float64 statistics of the exact convolution
    (bf16 operands, float64 sums) to the bf16 map the apply kernel reads, so the comparison measures the statistics path."""
    B, H, W, Cin, C = 2, 12, 20, 128, 256
    g = G(seed)
    x = torch.randn(B, H, W, Cin, generator=g).to(dev).bfloat16()
    w = (torch.randn(C, Cin, 1, 1, generator=g) / Cin ** 0.5).to(dev)
    bias = (ratio + 0.1 * torch.randn(C, generator=g)).to(dev)
    gw, gb = (1 + 0.3 * torch.randn(C, generator=g)).to(dev), (0.5 * torch.randn(C, generator=g)).to(dev)
    st = torch.zeros(B, G_, 2, dtype=torch.int64, device=dev)
    y = ops.conv2d(x, ops.pack_conv_weight(w), 1, 1, bias=bias, gn_stats=st, gn_groups=G_)
    pre = torch.einsum("bhwk,ck->bhwc", x.double(), w.bfloat16().double()[:, :, 0, 0]) + bias.double()
    pg = pre.reshape(B, H * W, G_, C // G_)
    mean, var = pg.mean((1, 3)), pg.var((1, 3), unbiased=False)
    worst = 0.0
    for act in ACT_REF:
        out = ops.groupnorm_apply(y, st, gw, gb, G_, eps, act, out=torch.empty_like(y))
        ref = gn_ref(y, mean, var, eps, gw, gb, act)
        worst = max(worst, ((out.double() - ref).abs() / (ref.abs() * REL[torch.bfloat16] + GN_FLOOR)).max().item())
    print(f"err/bound {worst:.3f}  conv->gn chain |mean|/std={ratio} G={G_} (realised {(mean.abs() / var.sqrt()).max().item():.0f})")
    return worst


@pytest.mark.parametrize("ratio", [0, 10, 100])
@pytest.mark.parametrize("G_,eps", [(16, 1e-3), (32, 1e-5)])
def test_conv_groupnorm_chain(ratio, G_, eps):
    """|mean| / std up to 100 holds to float64 within one bf16 rounding."""
    assert conv_gn_chain(ratio, G_, eps) <= 1.0


@pytest.mark.xfail(strict=True, reason="the statistics are one-pass fixed-point sums of fp32 partial sums and squares: at |mean| / std = "
                                      "1000 the variance E[x^2] - mean^2 keeps only a few correct bits (err / bound 2.5 on an H100 SXM at 700 W)")
def test_conv_groupnorm_chain_offset_1000():
    assert conv_gn_chain(1000, 16, 1e-3) <= 1.0


def test_groupnorm_apply_act_check_is_not_vacuous():
    """The same check with the reference of the wrong activation fails: SiLU output against the identity reference."""
    g = G(16)
    x = torch.randn(1, 4, 5, 64, generator=g).to(dev).bfloat16()
    gw, gb = torch.ones(64, device=dev), torch.zeros(64, device=dev)
    st = fixed_point_stats(x, 8)
    mean, var = moments(st, 4 * 5 * 8)
    out = ops.groupnorm_apply(x, st, gw, gb, 8, 1e-3, ops.ACT_SILU, out=torch.empty_like(x))
    with pytest.raises(AssertionError):
        check(out, gn_ref(x, mean, var, 1e-3, gw, gb, ops.ACT_NONE), REL[torch.bfloat16], GN_FLOOR, "silu vs identity (must fail)")


@pytest.mark.parametrize("act", [ops.ACT_GELU, ops.ACT_SIGMOID])
def test_groupnorm_apply_rejects_unimplemented_activation(act):
    """GELU and SIGMOID are not implemented by the apply kernel: the call raises and writes nothing (it used to return the
    un-activated result)."""
    x = torch.randn(1, 4, 5, 64, generator=G(17)).to(dev).bfloat16()
    st = fixed_point_stats(x, 8)
    out = torch.full_like(x, 3.0)
    with pytest.raises(UnicornB200Error, match="act must be"):
        ops.groupnorm_apply(x, st, torch.ones(64, device=dev), torch.zeros(64, device=dev), 8, 1e-3, act, out=out)
    torch.cuda.synchronize()
    assert (out == 3.0).all()


def test_groupnorm_apply_rejects_misaligned_slice():
    """A channel slice 4 elements into a buffer has legal strides but a base that is not 16-byte aligned: rejected before launch."""
    buf = torch.zeros(1, 4, 5, 72, device=dev, dtype=torch.bfloat16)
    st = torch.zeros(1, 8, 2, dtype=torch.int64, device=dev)
    with pytest.raises(UnicornB200Error, match="16-byte aligned"):
        ops.groupnorm_apply(buf[..., 4:68], st, torch.ones(64, device=dev), torch.zeros(64, device=dev), 8, 1e-3, ops.ACT_NONE)


# ---------------------------------------------------------------------------------------------------------------- LayerNorm
LN_FLOOR = 1e-3


def ln_rows(M, C, dtype, g):
    """Row 0 constant (the output must be the bias), rows 1 / 2 at |mean| / std = 1e3, the rest ordinary."""
    x = torch.randn(M, C, generator=g, dtype=torch.float64) * 2 + 0.5
    x[0] = 0.30078125
    if M > 2:
        x[1] = offset_values(C, 768.0, 1e3, dtype, g)
        x[2] = offset_values(C, -384.0, 1e3, dtype, g)
    return x.to(dev, dtype)


def ln_ref(v, w, b, eps):
    mean = v.mean(1, keepdim=True)
    var = ((v - mean) ** 2).mean(1, keepdim=True)
    return (v - mean) / (var + eps).sqrt() * w.double() + b.double()


def run_ln(C, dtype, lo, seed, name):
    """uc_layernorm on [M, C] views starting lo channels into wider buffers, with and without the residual input, M = 1 and M = 9
    (one full and one partial block of 8 rows).  The buffer widths (the row strides) are C + 16, C + 24 and C + 32, multiples of 8
    whenever C is: with lo = 2 the views are 4-byte but not 16-byte aligned and that base offset alone must select the 32-bit
    kernel."""
    g = G(seed)
    w, b = (1 + 0.3 * torch.randn(C, generator=g)).to(dev), torch.randn(C, generator=g).to(dev)
    for M in (1, 9):
        xb = torch.zeros(M, C + 16, device=dev, dtype=dtype)
        x = xb[:, lo:lo + C]
        x.copy_(ln_rows(M, C, dtype, g))
        rb = torch.zeros(M, C + 24, device=dev, dtype=dtype)
        res = rb[:, lo:lo + C]
        res.copy_((torch.randn(M, C, generator=g) * 0.5).to(dev, dtype))
        res[:3] = 0.0  # the constant row and the offset rows keep their statistics
        for r in (None, res):
            yb = torch.randn(M, C + 32, generator=g).to(dev, dtype)
            yb0 = yb.clone()
            y = yb[:, lo:lo + C]
            if C % 8 == 0:  # strides that the 128-bit kernel accepts: only the base pointers decide which kernel runs
                assert x.stride(0) % 8 == 0 and res.stride(0) % 8 == 0 and y.stride(0) % 8 == 0
                assert all((t.data_ptr() % 16 != 0) == (lo % 8 != 0) for t in (x, res, y))
            ops.layernorm(x, w, b, 1e-6, res=r, out=y)
            v = x.double() + (r.double() if r is not None else 0)
            ref = ln_ref(v, w, b, 1e-6)
            tag = f"{name} M={M} res={r is not None}"
            check(y, ref, REL[dtype], LN_FLOOR, tag)
            check(y[0], b.double(), REL[dtype], LN_FLOOR, tag + " constant row = bias")
            guards_kept(yb, yb0, lo, C, tag)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("C,lo", [(98, 0), (250, 0), (382, 0), (766, 0), (1534, 0), (2046, 0),
                                  (96, 2), (256, 2), (384, 2), (768, 2), (1536, 2), (2048, 2)])
def test_layernorm_32bit_kernel(C, lo, dtype):
    """Every layernorm_kernel<MAXI> (MAXI = 2, 4, 6, 12, 24, 32): C % 8 != 0, or C % 8 == 0 as a view that is not 16-byte aligned."""
    run_ln(C, dtype, lo, 20 + C, f"ln32 C={C} lo={lo} {dtype}")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("C", [96, 256, 512, 768, 1536, 2048])
def test_layernorm_v8_kernel(C, dtype):
    """Every layernorm_v8_kernel<MAXV> (MAXV = 1, 2, 3, 6, 8) on 16-byte aligned views."""
    run_ln(C, dtype, 8, 40 + C, f"ln v8 C={C} {dtype}")


# ---------------------------------------------------------------------------------------------------------------- correlation
# The output is fp32, so the relative term is not an output rounding: it covers the approximate exponentials (ex2.approx and the
# polynomial exp2, relative errors below 3e-6) with room to spare, and catches errors of 1e-4 and above in either dtype.
CORR_REL = 2.0 ** -14
CORR_FLOOR = 1e-6
# the similarities are fp32 sums of 128 exact products: a logit error of a few fp32 ulps of max|S| moves an output by up to that much
# times the spread of the values
CORR_LOGIT_ULPS = 2.0 ** -22


def run_corr(k, q, v, n_obj, dtype, name):
    """out[o, j] = sum_i v[o, i] softmax_i(<k_i, q_j>) with ld_ref, ld_cur > 128, ldv > n_ref, ldo > n_cur and guard rows
    n_obj..7 / guard columns around the output."""
    n_ref, n_cur = k.shape[0], q.shape[0]
    kb = torch.zeros(n_ref, 136, device=dev, dtype=dtype)
    kb[:, :128] = k.to(dtype)
    qb = torch.zeros(n_cur, 200, device=dev, dtype=dtype)
    qb[:, 8:136] = q.to(dtype)
    vb = torch.zeros(n_obj, n_ref + 5, device=dev)
    vb[:, :n_ref] = v
    ob = torch.full((8, n_cur + 3), 1234.5, device=dev)
    ops.corr_propagate(kb[:, :128], qb[:, 8:136], vb[:, :n_ref], out=ob[:n_obj, :n_cur])
    S = kb[:, :128].double() @ qb[:, 8:136].double().t()
    ref = v.double() @ torch.softmax(S, dim=0)
    floor = CORR_FLOOR + CORR_LOGIT_ULPS * S.abs().max().item() * v.abs().max().item()
    r = check(ob[:n_obj, :n_cur], ref, CORR_REL, floor, name)
    assert (ob[n_obj:] == 1234.5).all() and (ob[:, n_cur:] == 1234.5).all(), f"{name}: guard rows / columns of out overwritten"
    return r


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("n_obj", range(1, 9))
def test_corr_propagate_sizes(n_obj, dtype):
    """NOBJ = 1, 2, 4, 8 kernels with every n_obj they serve, tail chunks (n_ref 1, 127..129, 1000) and tail tiles (n_cur 1, 129)."""
    g = G(30 + n_obj)
    for n_ref in (1, 127, 128, 129, 1000):
        for n_cur in (1, 129):
            k = torch.randn(n_ref, 128, generator=g) * 0.5
            q = torch.randn(n_cur, 128, generator=g) * 0.5
            v = torch.rand(n_obj, n_ref, generator=g)
            run_corr(k.to(dev), q.to(dev), v.to(dev), n_obj, dtype, f"corr n_obj={n_obj} n_ref={n_ref} n_cur={n_cur} {dtype}")


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("n_obj", [1, 2, 5, 8])
def test_corr_propagate_hard_softmax(n_obj, dtype):
    """Near one-hot softmax: similarities spanning about +-300 (most exponents far below the -125 clamp of the polynomial exp2), and
    keys ordered by similarity so that every chunk raises the running maximum and the largest one arrives in the last chunk."""
    g = G(50 + n_obj)
    n_ref, n_cur = 1000, 129
    u = torch.randn(128, generator=g)
    u = u / u.norm()
    # random keys and queries with |<k, q>| up to ~300
    k = torch.randn(n_ref, 128, generator=g) * 3.0
    q = torch.randn(n_cur, 128, generator=g) * 3.0
    v = torch.rand(n_obj, n_ref, generator=g)
    run_corr(k.to(dev), q.to(dev), v.to(dev), n_obj, dtype, f"corr +-300 n_obj={n_obj} {dtype}")
    # keys along u with increasing weight, queries along u: s_ij increases with i for every j, the maximum is key n_ref - 1
    beta = torch.linspace(-1.0, 1.0, n_ref)[:, None]
    k2 = beta * u * 17.0 + 0.05 * torch.randn(n_ref, 128, generator=g)
    q2 = u * 17.0 * (1 + 0.2 * torch.rand(n_cur, 1, generator=g)) + 0.05 * torch.randn(n_cur, 128, generator=g)
    S = k2.to(dtype).double() @ q2.to(dtype).double().t()
    assert (S.argmax(0) >= 896).all() and S.max().item() > 250
    run_corr(k2.to(dev), q2.to(dev), v.to(dev), n_obj, dtype, f"corr max in last chunk n_obj={n_obj} {dtype}")


# ---------------------------------------------------------------------------------------------------------------- small kernels
@pytest.mark.parametrize("C0", [32, 64, 96, 128, 192, 256])
def test_stem_ln_channel_counts(C0):
    """stem_ln_kernel<CPL> for CPL = 1, 2, 3, 4, 6, 8; W / 4 = 9 leaves a partial group of 4 output pixels per row."""
    g = G(60 + C0)
    img = (torch.rand(2, 3, 24, 36, generator=g) * 255).to(dev)
    w = (torch.randn(C0, 3, 4, 4, generator=g) / 7).to(dev)
    b, lw, lb = (torch.randn(C0, generator=g).to(dev) for _ in range(3))
    out = ops.stem_ln(img, ops.pack_stem_weight(w), b, lw, lb)
    x = F.conv2d(img.double(), w.double(), b.double(), stride=4).permute(0, 2, 3, 1)
    ref = F.layer_norm(x, (C0,), lw.double(), lb.double(), 1e-6)
    check(out, ref, REL[torch.bfloat16], 1e-3, f"stem C0={C0}")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_copy_upsample_plain_copy(dtype):
    """up = 1: a slice-to-slice copy, exact, guard columns of both buffers untouched."""
    src_b, src = guarded((2, 5, 7), 40, 8, 16, dtype, 70)
    dst_b, dst = guarded((2, 5, 7), 40, 24, 8, dtype, 71)
    src0, dst0 = src_b.clone(), dst_b.clone()
    ops.copy_upsample(src, dst, 1)
    assert torch.equal(dst, src) and torch.equal(src_b, src0)
    guards_kept(dst_b, dst0, 24, 40, "copy_upsample up=1")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_add_strided(dtype):
    """y = a + b with one rounding, on strided rows and into a slice of a wider buffer."""
    g = G(72)
    M, C = 37, 48
    a = torch.randn(M, C + 16, generator=g).to(dev, dtype)[:, 8:8 + C]
    b = (torch.randn(M, C + 8, generator=g) * 3).to(dev, dtype)[:, :C]
    yb, y = guarded((M,), C, 16, 8, dtype, 73)
    y0 = yb.clone()
    ops.add(a, b, out=y)
    assert torch.equal(y, (a.double() + b.double()).to(dtype))
    guards_kept(yb, y0, 16, C, "add")

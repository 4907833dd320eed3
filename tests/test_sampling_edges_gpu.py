"""Edge-case parity of the kernels that read a feature map at a computed position against float64 references on the same rounded
operands: the deformable attention (uc_msda_fused_bf16 / _batched, uc_msda_forward_f32), the MOT embedding sampler
(uc_sample_embed / _batched), the bi-softmax association scores (uc_bisoftmax), the mask branch's aligned-bilinear fusion
(uc_aligned_bilinear_add / _batched), the CondInst mask head (uc_dynamic_masks / _batched) and the fp32 bilinear resize
(uc_bilinear_f32).  Samples sit on pixel centres, in the bands (-1, 0) and (H-1, H), exactly on -1 and H and far outside; maps are
1 or 2 pixels wide; levels have distinct sizes; strides, counts and batch layouts leave padding, tails and skipped images that
must stay untouched.

Each reference is a plain float64 restatement (explicit four-tap bilinear sampling, explicit softmax, explicit 1x1 layers) on the
kernel's rounded operands.  Positions are the one exception: they are computed with the fp32 arithmetic the reference model uses,
and where the kernel may contract or reorder that arithmetic the bound has a position term (a few fp32 ulps of the coordinate x
twice the largest value of the sampled map x the sample weight).  The CPU tests pin every float64 reference to the existing
definition (grid_sample, the oracles, F.interpolate) to 1e-12 on the same float64 positions.

Bounds are per element: |got - ref| <= bound, with bf16 outputs at 2^-8 |ref| (one rounding to bf16) and every output at
k * 2^-24 * sum|terms| (fp32 accumulation; sum|terms| from a second float64 pass on absolute values), plus the terms derived in each
test's docstring and a floor of 1e-7 max|ref|.  Every check prints its largest err / bound, and the checks that could pass by
accident also run against a deliberately wrong reference, where they must fail."""
import ctypes
import os
import sys

import pytest
import torch
import torch.nn.functional as F

from unicorn_b200 import ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import tracker_oracle  # noqa: E402
import unicorn_oracle as orc  # noqa: E402
from test_kernels_gpu import _msda_ref  # noqa: E402
from test_launch_parity_gpu import msda_reference  # noqa: E402

gpu = pytest.mark.gpu
dev = "cuda"
f64 = torch.float64
REL = 2.0 ** -8   # one rounding to bf16
U = 2.0 ** -24    # fp32 unit roundoff
FLOOR = 1e-7      # x max|ref|
SELF_TOL = 1e-12  # float64 reference vs the existing definition


def G(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def check(got, ref, bound, name):
    """Per-element |got - ref| <= bound; ref and bound float64."""
    err = (got.double() - ref).abs()
    ratio = (err / bound).max().item() if err.numel() else 0.0
    print(f"err/bound {ratio:.3f}  {name}")
    assert ratio <= 1.0, f"{name}: max err/bound {ratio:.3g} (max err {err.max().item():.3g})"
    return ratio


def floor_of(ref):
    return FLOOR * ref.abs().max().item() + 1e-300


def self_check(a, b, name):
    err = (a - b).abs().max().item() if a.numel() else 0.0
    print(f"self-check {err:.2e}  {name}")
    assert err <= SELF_TOL, f"{name}: float64 reference differs from the existing definition by {err:.3g}"


def must_fail(fn):
    with pytest.raises(AssertionError):
        fn()


def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def edge_coords(n, size, g):
    """n float64 pixel coordinates along an axis of `size` pixels (h_im = loc * size - 0.5): random in (-1.5, size + 0.5), on a
    pixel centre, in the band (-1, 0), in the band (size - 1, size), exactly -1, exactly size, or far outside on either side."""
    cat = torch.randint(0, 8, (n,), generator=g)
    u = torch.rand(n, generator=g, dtype=f64).clamp(1e-3, 1 - 1e-3)
    side = torch.rand(n, generator=g) < 0.5
    far = torch.where(side, -3.0 - 40 * u, size + 2.0 + 40 * u)
    opts = [-1.5 + (size + 2.0) * u, torch.floor(u * size), -1.0 + u, size - 1.0 + u, torch.full_like(u, -1.0),
            torch.full_like(u, float(size)), far, -1.5 + (size + 2.0) * u]
    c = torch.empty(n, dtype=f64)
    for k, o in enumerate(opts):
        c[cat == k] = o[cat == k]
    return c


# ================================================================================================ deformable attention
def msda_ref(value, hw, loc, attn, swap=False):
    """float64 deformable attention (ms_deformable_im2col, the CUDA operator's form): value [N, S, M, D], loc [N, Lq, M, L, P, 2]
    normalised (x, y), attn [N, Lq, M, L, P] -> [N, Lq, M, D].  h_im = loc_y * H - 0.5, w_im = loc_x * W - 0.5; a sample counts only
    if -1 < h_im < H and -1 < w_im < W; each of its four corners that lies in the map adds its bilinear weight x value.  swap=True
    exchanges the weights of the (0, 1) and (1, 0) corners (a wrong reference)."""
    N, S, M, D = value.shape
    Lq = loc.shape[1]
    out = torch.zeros(N, Lq, M, D, dtype=f64, device=value.device)
    n_i = torch.arange(N, device=value.device)[:, None, None, None]
    m_i = torch.arange(M, device=value.device)[None, None, :, None]
    start = 0
    for l, (H, W) in enumerate(hw):
        v = value[:, start:start + H * W]
        start += H * W
        x = loc[:, :, :, l, :, 0].double() * W - 0.5
        y = loc[:, :, :, l, :, 1].double() * H - 0.5
        ok = (y > -1) & (x > -1) & (y < H) & (x < W)
        y0, x0 = torch.floor(y), torch.floor(x)
        ly, lx = y - y0, x - x0
        w01, w10 = (1 - ly) * lx, ly * (1 - lx)
        if swap:
            w01, w10 = w10, w01
        a = attn[:, :, :, l].double()
        for dy, dx, wt in ((0, 0, (1 - ly) * (1 - lx)), (0, 1, w01), (1, 0, w10), (1, 1, ly * lx)):
            yy, xx = y0 + dy, x0 + dx
            inb = ok & (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
            idx = (yy.clamp(0, H - 1) * W + xx.clamp(0, W - 1)).long()
            out += ((wt * inb * a)[..., None] * v[n_i, idx, m_i]).sum(3)
    return out


def msda_pos_term(value, hw, loc, attn, ulps):
    """Position term: a coordinate off by `ulps` fp32 ulps of (|coordinate| + 1) moves a bilinear sample by at most that distance x
    its largest adjacent tap difference <= 2 max|v| of the level; summed over the samples near the map with their weights."""
    out = torch.zeros(value.shape[0], loc.shape[1], value.shape[2], value.shape[3], dtype=f64, device=value.device)
    start = 0
    for l, (H, W) in enumerate(hw):
        vmax = value[:, start:start + H * W].abs().amax(1)  # [N, M, D]
        start += H * W
        x = loc[:, :, :, l, :, 0].double() * W - 0.5
        y = loc[:, :, :, l, :, 1].double() * H - 0.5
        near = (y > -2) & (x > -2) & (y < H + 1) & (x < W + 1)
        d = ulps * U * (x.abs() + y.abs() + 2)
        out += (attn[:, :, :, l].double().abs() * d * near).sum(-1)[..., None] * 2 * vmax[:, None]
    return out


def fused_rows(hw, B):
    """row[b, q]: the row of query q (the levels' pixel grids, concatenated) of image b in ops.msda_fused's level-major layout
    (level l of image b starts at row B * start_l + b * h_l * w_l)."""
    Lq = sum(h * w for h, w in hw)
    row = torch.empty(B, Lq, dtype=torch.long)
    q0 = 0
    for H, W in hw:
        for b in range(B):
            row[b, q0:q0 + H * W] = B * q0 + b * H * W + torch.arange(H * W)
        q0 += H * W
    return row


def fused_refpts(hw):
    """Reference point of every query, fp32 as the model computes it: ((qx + 0.5) / Wq, (qy + 0.5) / Hq); and each query's level."""
    rx, ry, ql = [], [], []
    for l, (H, W) in enumerate(hw):
        qi = torch.arange(H * W)
        rx.append(((qi % W).float() + 0.5) / W)
        ry.append(((qi // W).float() + 0.5) / H)
        ql.append(torch.full((H * W,), l))
    return torch.cat(rx), torch.cat(ry), torch.cat(ql)


def fused_inputs(offlog, hw, B, M, P, norm="sampled"):
    """Per-image sampling locations [B, Lq, M, L, P, 2] and logits [B, Lq, M, L*P] of uc_msda_fused from its offlog rows: loc = r +
    off / (W, H) of the sampled level, in offlog's dtype (fp32: the model's own arithmetic).  norm="query" normalises by the query
    level's size instead (a wrong reference)."""
    L = len(hw)
    LP = L * P
    row = fused_rows(hw, B).to(offlog.device)
    Lq = row.shape[1]
    rx, ry, ql = (t.to(offlog.device) for t in fused_refpts(hw))
    rows = offlog[row]
    off = rows[..., :M * LP * 2].reshape(B, Lq, M, L, P, 2)
    lg = rows[..., M * LP * 2:M * LP * 3].reshape(B, Lq, M, LP)
    Ws = torch.tensor([w for _, w in hw], dtype=offlog.dtype, device=offlog.device)
    Hs = torch.tensor([h for h, _ in hw], dtype=offlog.dtype, device=offlog.device)
    if norm == "query":
        Wn, Hn = Ws[ql][None, :, None, None, None], Hs[ql][None, :, None, None, None]
    else:
        Wn, Hn = Ws[None, None, None, :, None], Hs[None, None, None, :, None]
    lx = rx.to(offlog.dtype)[None, :, None, None, None] + off[..., 0] / Wn
    ly = ry.to(offlog.dtype)[None, :, None, None, None] + off[..., 1] / Hn
    return torch.stack([lx, ly], -1), lg


def softmax64(lg):
    x = lg.double() - lg.double().amax(-1, keepdim=True)
    e = torch.exp(x)
    return e / e.sum(-1, keepdim=True), x


def fused_reference(value, offlog, hw, B, M, P, norm="sampled"):
    """float64 output of uc_msda_fused per image [B, Lq, M*32], and the bound.
    Bound: 2^-8 |ref| + (4 + 4 L P) 2^-24 S + E + X + floor, where
      S  = the same sum on |v| (each corner weight hh * hw * a is rounded at most 4 times, and each of the 4 L P corner FMAs rounds
           the partial sum once);
      E  = sum over the samples of |v| x a_i x (e_i + sum_j a_j e_j + (L P + 2) 2^-24): __expf(x) is within 2 + 1.173 |x| ulps
           (2^-23 relative each, CUDA programming guide), x = logit - max rounds once more (|x| 2^-24), the denominator adds L P
           roundings, 1 / den and the product one each;
      X  = the position term with 5 ulps (r + off / W rounds 3 times in the model too; the kernel may contract ly * H - 0.5)."""
    L = len(hw)
    loc, lg = fused_inputs(offlog, hw, B, M, P, norm)
    a, x = softmax64(lg)
    e = (2 + 1.173 * x.abs()) * 2.0 ** -23 + x.abs() * U
    rel = e + (a * e).sum(-1, keepdim=True) + (L * P + 2) * U
    Lq = loc.shape[1]
    shape = (B, Lq, M, L, P)
    v = value.double()[fused_rows(hw, B).to(value.device)].reshape(B, Lq, M, 32)
    ref = msda_ref(v, hw, loc, a.reshape(shape))
    S = msda_ref(v.abs(), hw, loc, a.reshape(shape))
    E = msda_ref(v.abs(), hw, loc, (a * rel).reshape(shape))
    X = msda_pos_term(v, hw, loc, a.reshape(shape), 5)
    bound = REL * ref.abs() + (4 + 4 * L * P) * U * S + E + X
    bound = bound + floor_of(ref)
    return ref.reshape(B, Lq, M * 32), bound.reshape(B, Lq, M * 32)


def fused_case(hw, B, M, P, seed, ld_pad=5, device=dev):
    """value bf16 [B*Lq, M*32] (different content per image); offlog fp32 rows of ld = M L P 3 + ld_pad whose padding columns are
    NaN; offsets that put every sample on one of edge_coords' categories of the sampled level (x and y independently); logits in
    two regimes: comparable weights (std 2) for half the (query, head) pairs, a range of 80 with one dominant +40 for the rest."""
    g = G(seed)
    L, Lq = len(hw), sum(h * w for h, w in hw)
    LP = L * P
    rows = B * Lq
    value = torch.randn(rows, M * 32, generator=g).bfloat16()
    ld = M * LP * 3 + ld_pad
    offlog = torch.full((rows, ld), float("nan"))
    rx, ry, _ = fused_refpts(hw)
    row = fused_rows(hw, B)
    off = torch.empty(B, Lq, M, L, P, 2, dtype=f64)
    n = B * Lq * M * P
    for l, (H, W) in enumerate(hw):
        cx = edge_coords(n, W, g).reshape(B, Lq, M, P)
        cy = edge_coords(n, H, g).reshape(B, Lq, M, P)
        off[:, :, :, l, :, 0] = cx + 0.5 - rx.double()[None, :, None, None] * W
        off[:, :, :, l, :, 1] = cy + 0.5 - ry.double()[None, :, None, None] * H
    lg = torch.randn(B, Lq, M, LP, generator=g, dtype=f64) * 2
    hot = torch.rand(B, Lq, M, generator=g) < 0.5
    wide = torch.rand(B, Lq, M, LP, generator=g, dtype=f64) * 80 - 40
    wide.scatter_(-1, torch.randint(0, LP, (B, Lq, M, 1), generator=g), 40.0)
    lg = torch.where(hot[..., None], wide, lg)
    body = torch.cat([off.reshape(B, Lq, -1), lg.reshape(B, Lq, -1)], -1).float()
    offlog[row.reshape(-1), :M * LP * 3] = body.reshape(rows, -1)
    return value.to(device), offlog.to(device)


def run_fused(value, offlog, hw, M, P, sentinel=-777.0):
    """ops.msda_fused into the prefix of a larger bf16 buffer filled with a sentinel; returns (out, tail)."""
    n = value.shape[0] * M * 32
    buf = torch.full((n + 7 * M * 32 + 3,), sentinel, dtype=torch.bfloat16, device=dev)
    out = buf[:n].view(value.shape[0], M * 32)
    offv = offlog[:, :M * len(hw) * P * 3]
    assert offv.stride(0) == offlog.shape[1]
    ops.msda_fused(value, offv, hw, M, P, out=out)
    torch.cuda.synchronize()
    return out, buf[n:]


LV1 = [(6, 5)]
LV2 = [(8, 4), (3, 7)]
LV3 = [(1, 1), (1, 16), (8, 1)]
LV4 = [(4, 8), (1, 1), (1, 7), (5, 1)]
FUSED_CASES = [(LV1, 1, 1, 1), (LV1, 16, 8, 1), (LV2, 8, 8, 1), (LV3, 5, 8, 1), (LV4, 4, 1, 1), (LV4, 4, 8, 1),
               (LV4, 4, 8, 2), (LV2, 8, 8, 3), (LV3, 5, 1, 4), (LV1, 16, 1, 4)]


@gpu
@pytest.mark.parametrize("hw,P,M,B", FUSED_CASES)
def test_msda_fused_edges(hw, P, M, B):
    """uc_msda_fused_bf16 (B = 1) and _batched: every sample on an edge category, distinct level sizes with 1x1, 1xW and Hx1
    levels, NaN padding columns in offlog (never read), and the output as the prefix of a sentinel buffer (no row past B*Lq written).
    Bound: fused_reference."""
    value, offlog = fused_case(hw, B, M, P, 1000 + 10 * B + M + P)
    out, tail = run_fused(value, offlog, hw, M, P)
    assert bool((tail == -777.0).all()), "uc_msda_fused wrote past its B*Lq output rows"
    ref, bound = fused_reference(value, offlog, hw, B, M, P)
    got = out[fused_rows(hw, B).to(dev)]
    check(got, ref, bound, f"msda fused hw={hw} P={P} M={M} B={B}")


@gpu
@pytest.mark.parametrize("hw,B", [((20, 20), 1), ((20, 20), 4), ((50, 80), 1), ((50, 80), 3)])
def test_msda_fused_production(hw, B):
    """The encoder's launch: two levels of the (h, w) the interaction sees (stride 16 of a 320x320 or 800x1280 input), M = 8,
    P = 4, B images.  Offsets N(0, 3^2) px and N(0, 1) logits as in test_kernels_gpu.  Bound: fused_reference."""
    g = G(11 + B)
    lv = [hw, hw]
    M, P, Lq = 8, 4, 2 * hw[0] * hw[1]
    value = torch.randn(B * Lq, 256, generator=g).bfloat16().to(dev)
    offlog = torch.cat([torch.randn(B * Lq, 128, generator=g) * 3, torch.randn(B * Lq, 64, generator=g)], 1).to(dev)
    out, tail = run_fused(value, offlog, lv, M, P)
    assert bool((tail == -777.0).all())
    ref, bound = fused_reference(value, offlog, lv, B, M, P)
    check(out[fused_rows(lv, B).to(dev)], ref, bound, f"msda fused production hw={hw} B={B}")


@gpu
def test_msda_fused_checks_are_not_vacuous():
    """The fused check tells the sampled level's size from the query level's (offsets normalised by lv.W[ql]) and notices a half-pixel
    shift of the sampling grid."""
    hw, P, M, B = LV4, 4, 8, 2
    value, offlog = fused_case(hw, B, M, P, 1000 + 10 * B + M + P)
    out, _ = run_fused(value, offlog, hw, M, P)
    got = out[fused_rows(hw, B).to(dev)]
    ref, bound = fused_reference(value, offlog, hw, B, M, P, norm="query")
    must_fail(lambda: check(got, ref, bound, "msda fused vs the query level's W (must fail)"))
    shifted = offlog.clone()
    shifted[:, :M * len(hw) * P * 2] += 0.5
    ref, bound = fused_reference(value, shifted, hw, B, M, P)
    must_fail(lambda: check(got, ref, bound, "msda fused vs a half-pixel shift (must fail)"))


def f32_case(B, Lq, M, D, hw, P, seed):
    g = G(seed)
    L = len(hw)
    S = sum(h * w for h, w in hw)
    value = torch.randn(B, S, M, D, generator=g)
    loc = torch.empty(B, Lq, M, L, P, 2, dtype=f64)
    n = B * Lq * M * P
    for l, (H, W) in enumerate(hw):
        loc[:, :, :, l, :, 0] = ((edge_coords(n, W, g) + 0.5) / W).reshape(B, Lq, M, P)
        loc[:, :, :, l, :, 1] = ((edge_coords(n, H, g) + 0.5) / H).reshape(B, Lq, M, P)
    attn = torch.softmax(torch.randn(B, Lq, M, L * P, generator=g) * 2, -1).reshape(B, Lq, M, L, P)
    shapes = torch.tensor(hw, dtype=torch.long)
    lsi = torch.cat([shapes.new_zeros(1), shapes.prod(1).cumsum(0)[:-1]])
    return [t.to(dev) for t in (value, shapes, lsi, loc.float(), attn)]


def f32_bound(value, hw, loc, attn, ref):
    """uc_msda_forward_f32: per sample hh, hw, the two products and v (4 roundings per corner), the 3-term corner sum, x a and the
    accumulation: (9 + L P) 2^-24 S, S the same sum on |v|; the position term with 3 ulps (the kernel may contract loc * H - 0.5)."""
    L, P = loc.shape[3], loc.shape[4]
    S = msda_ref(value.double().abs(), hw, loc, attn)
    X = msda_pos_term(value.double(), hw, loc, attn, 3)
    return (9 + L * P) * U * S + X + floor_of(ref)


F32_HW = [(6, 5), (1, 1), (1, 9), (4, 1)]


@gpu
@pytest.mark.parametrize("B,Lq,M,D", [(2, 7, 3, 1), (2, 29, 2, 3), (2, 50, 2, 32), (2, 13, 3, 33), (2, 5000, 8, 32)])
def test_msda_f32_edges(B, Lq, M, D):
    """uc_msda_forward_f32 with D = 1, 3, 32, 33, four levels of distinct shapes (1x1, 1xW, Hx1), Lq != S, B = 2, every sample on
    an edge category; the last case has B Lq M D > num_sms * 32 * 256, so the capped grid-stride loop runs several times."""
    value, shapes, lsi, loc, attn = f32_case(B, Lq, M, D, F32_HW, 4, 2000 + Lq + D)
    if Lq == 5000:
        assert B * Lq * M * D > num_sms() * 32 * 256
    out = ops.msda_forward(value, shapes, lsi, loc, attn)
    ref = msda_ref(value.double(), F32_HW, loc, attn).reshape(B, Lq, M * D)
    bound = f32_bound(value, F32_HW, loc, attn, ref).reshape(B, Lq, M * D)
    check(out, ref, bound, f"msda f32 B={B} Lq={Lq} M={M} D={D}")


@gpu
def test_msda_f32_checks_are_not_vacuous():
    """The f32 check notices the (0, 1) and (1, 0) corner weights swapped."""
    value, shapes, lsi, loc, attn = f32_case(2, 50, 2, 32, F32_HW, 4, 2082)
    out = ops.msda_forward(value, shapes, lsi, loc, attn)
    ref = msda_ref(value.double(), F32_HW, loc, attn, swap=True).reshape(2, 50, 64)
    bound = f32_bound(value, F32_HW, loc, attn, ref).reshape(2, 50, 64)
    must_fail(lambda: check(out, ref, bound, "msda f32 vs swapped corner weights (must fail)"))


def test_msda_reference_matches_grid_sample():
    """msda_ref equals _msda_ref (F.grid_sample, zeros, align_corners=False) in float64 on the same locations, with samples on every
    edge category of four distinct levels; and the fused reference's layout, reference points and softmax equal msda_reference
    (which accumulates in fp32, so to 1e-6 of max|ref| there)."""
    g = G(5)
    B, Lq, M, D, P = 2, 23, 3, 4, 3
    hw = F32_HW
    S = sum(h * w for h, w in hw)
    value = torch.randn(B, S, M, D, generator=g, dtype=f64)
    loc = torch.empty(B, Lq, M, len(hw), P, 2, dtype=f64)
    for l, (H, W) in enumerate(hw):
        loc[:, :, :, l, :, 0] = ((edge_coords(B * Lq * M * P, W, g) + 0.5) / W).reshape(B, Lq, M, P)
        loc[:, :, :, l, :, 1] = ((edge_coords(B * Lq * M * P, H, g) + 0.5) / H).reshape(B, Lq, M, P)
    attn = torch.rand(B, Lq, M, len(hw), P, generator=g, dtype=f64)
    self_check(msda_ref(value, hw, loc, attn).reshape(B, Lq, M * D), _msda_ref(value, hw, loc, attn), "msda vs grid_sample")
    for hw in (LV4, LV3):
        M, P = 2, 4
        value, offlog = fused_case(hw, 1, M, P, 6, device="cpu")
        offlog = offlog.double()
        loc, lg = fused_inputs(offlog, hw, 1, M, P)
        a = softmax64(lg)[0].reshape(loc.shape[:-1])
        v = value.double().reshape(1, -1, M, 32)
        mine = msda_ref(v, hw, loc, a).reshape(-1, M * 32)
        self_check(mine, _msda_ref(v.reshape(1, -1, M, 32), hw, loc[0][None], a[0][None])[0], f"msda fused vs grid_sample hw={hw}")
        # msda_reference accumulates in fp32 (torch.zeros default dtype): its layout, reference points and softmax agree to fp32
        want = msda_reference(v[0].reshape(-1, M * 32), offlog, hw, M, P)
        err = (mine - want).abs().max().item()
        print(f"self-check {err:.2e}  msda fused vs msda_reference hw={hw} (fp32 accumulation)")
        assert err <= 1e-6 * mine.abs().max().item()


# ================================================================================================ embedding sampling
def embed_positions(boxes, h, w, s=8.0):
    """The sampling position (x, y) in map pixels of each box (rows x1, y1, x2, y2): tracker_oracle.sample_embeddings' centre
    expressions, then grid_sample's unnormalise ((c + 1) w - 1) / 2 and border clip, in the boxes' dtype."""
    cx = (boxes[:, 0] + boxes[:, 2]) / 2 / s - 0.5
    cy = (boxes[:, 1] + boxes[:, 3]) / 2 / s - 0.5
    cx = (torch.clamp(cx, min=0, max=w - 1) / (w - 1) - 0.5) * 2.0
    cy = (torch.clamp(cy, min=0, max=h - 1) / (h - 1) - 0.5) * 2.0
    x = ((cx + 1) * w - 1) / 2
    y = ((cy + 1) * h - 1) / 2
    return torch.clamp(x, 0, w - 1), torch.clamp(y, 0, h - 1)


def embed_ref(emb, x, y, swap=False):
    """float64 border-padded bilinear sample of emb [h, w, C] at (x, y) (float64, inside [0, w-1] x [0, h-1]) -> [n, C]: x0 =
    floor(x), x1 = min(x0 + 1, w - 1).  swap=True exchanges the weights of the (y0, x1) and (y1, x0) taps (a wrong reference)."""
    h, w = emb.shape[:2]
    x, y = x.double(), y.double()
    x0, y0 = torch.floor(x).long(), torch.floor(y).long()
    x1, y1 = (x0 + 1).clamp(max=w - 1), (y0 + 1).clamp(max=h - 1)
    lx, ly = (x - x0)[:, None], (y - y0)[:, None]
    w01, w10 = lx * (1 - ly), (1 - lx) * ly
    if swap:
        w01, w10 = w10, w01
    e = emb.double()
    return (1 - lx) * (1 - ly) * e[y0, x0] + w01 * e[y0, x1] + w10 * e[y1, x0] + lx * ly * e[y1, x1]


def embed_bound(emb, x, y, ref):
    """fp32 result: 1 - l, the weight products, the tap products and three adds: 6 2^-24 S (S on |v|); position term with 4 ulps of
    (x + y + 2) x 2 max|v| of the channel (the kernel may contract (c + 1) * w - 1)."""
    S = embed_ref(emb.abs(), x, y)
    vmax = emb.double().abs().amax((0, 1))
    X = 4 * U * (x.double() + y.double() + 2)[:, None] * 2 * vmax[None]
    return 6 * U * S + X + floor_of(ref)


def embed_boxes(n, h, w, g, s=8.0, ldb=7):
    """n box rows of ldb columns whose centres clamp on each side, lie exactly on the last row / column or on a pixel centre, or
    are random; the centre pixel is (x1 + x2) / 2 / s - 0.5."""
    cat = torch.randint(0, 7, (n,), generator=g)
    u, v = torch.rand(n, generator=g, dtype=f64), torch.rand(n, generator=g, dtype=f64)
    px = -1.5 + (w + 2) * u
    py = -1.5 + (h + 2) * v
    px = torch.where(cat == 0, -0.5 - 5 * u, px)                      # clamps left
    px = torch.where(cat == 1, w - 1 + 0.25 + 5 * u, px)              # clamps right
    py = torch.where(cat == 2, -0.5 - 5 * v, py)                      # clamps top
    py = torch.where(cat == 3, h - 1 + 0.25 + 5 * v, py)              # clamps bottom
    px = torch.where(cat == 4, float(w - 1), px)                      # last column / row exactly
    py = torch.where(cat == 4, float(h - 1), py)
    px = torch.where(cat == 5, torch.floor(u * w), px)                # pixel centres
    py = torch.where(cat == 5, torch.floor(v * h), py)
    X, Y = (px + 0.5) * s, (py + 0.5) * s
    bw, bh = torch.randint(1, 40, (n,), generator=g).double() * 2, torch.randint(1, 40, (n,), generator=g).double() * 2
    b = torch.rand(n, ldb, generator=g) * 100
    b[:, 0], b[:, 1], b[:, 2], b[:, 3] = (X - bw / 2).float(), (Y - bh / 2).float(), (X + bw / 2).float(), (Y + bh / 2).float()
    return b


def run_sample_embed(emb, ld, h, w, C, boxes, count, n_max, B=1, bs_embed=0, bs_boxes=0, bs_out=0, ldb=7, sentinel=-555.0):
    """The C entry points directly (channel slices and per-image strides the NHWC wrapper does not express)."""
    out = torch.full((max(B * max(bs_out, n_max * C), 1) + 17,), sentinel, device=dev)
    dt = ops._DT[emb.dtype]
    cnt = None if count is None else torch.tensor(count, dtype=torch.int32, device=dev)
    if B == 1:
        ops._lib.check(ops._L().uc_sample_embed(ops._p(emb), ld, h, w, C, dt, ops._p(boxes), ldb, ops._p(cnt), n_max,
                                                ctypes.c_float(8.0), ops._p(out), ops._S()), "uc_sample_embed")
    else:
        ops._lib.check(ops._L().uc_sample_embed_batched(ops._p(emb), ld, ctypes.c_long(bs_embed), h, w, C, dt, ops._p(boxes),
                                                        ldb, ctypes.c_long(bs_boxes), ops._p(cnt), n_max, ctypes.c_float(8.0),
                                                        ops._p(out), ctypes.c_long(bs_out), B, ops._S()), "uc_sample_embed_batched")
    torch.cuda.synchronize()
    return out


EMBED_MAPS = [(2, 5, 1, 3), (7, 2, 33, 40), (2, 2, 33, 33), (13, 21, 128, 160), (20, 36, 128, 128)]


@gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("h,w,C,ld", EMBED_MAPS)
def test_sample_embed_edges(h, w, C, ld, dtype):
    """uc_sample_embed on 2-pixel and non-square maps, C = 1, 33, 128 as a channel slice of a wider map (ld > C), dets rows of 7
    columns, centres that clamp on each side, lie on the last row / column or on a pixel centre; n_max in {1, 7, 8, 9, 300} (8 boxes
    per CTA) with count 0, below and above n_max: rows past min(count, n_max) keep their sentinel.  Bound: embed_bound."""
    g = G(3000 + h * w + C)
    full = torch.randn(h, w, ld, generator=g).to(dtype).to(dev)
    emb = full[..., :C]
    for n_max in (1, 7, 8, 9, 300):
        boxes = embed_boxes(n_max, h, w, g).to(dev)
        x, y = embed_positions(boxes[:, :4].float(), h, w)
        ref = embed_ref(emb, x, y)
        bound = embed_bound(emb, x, y, ref)
        for count in sorted({0, max(n_max - 3, 1) if n_max > 1 else 0, n_max + 4}):
            out = run_sample_embed(full, ld, h, w, C, boxes, [count], n_max)
            n = min(count, n_max)
            got = out[:n * C].view(n, C)
            check(got, ref[:n], bound[:n], f"sample_embed {dtype} h={h} w={w} C={C} ld={ld} n_max={n_max} count={count}")
            assert bool((out[n * C:] == -555.0).all()), "rows past the count were written"


@gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_sample_embed_batched_edges(dtype):
    """uc_sample_embed_batched: B = 3 images with distinct content and counts (below, above n_max, zero), per-image strides of the
    map, the boxes and the output larger than one image; every row past an image's count keeps its sentinel."""
    g = G(3100)
    B, h, w, C, ld, n_max = 3, 7, 11, 33, 36, 9
    bs_e, bs_b, bs_o = h * w * ld + 40, n_max * 7 + 13, n_max * C + 5
    emb_buf = torch.randn(B * bs_e, generator=g).to(dtype).to(dev)
    box_buf = torch.zeros(B * bs_b, device=dev)
    counts = [4, n_max + 3, 0]
    for b in range(B):
        box_buf[b * bs_b:b * bs_b + n_max * 7] = embed_boxes(n_max, h, w, g).reshape(-1).to(dev)
    out = run_sample_embed(emb_buf, ld, h, w, C, box_buf, counts, n_max, B, bs_e, bs_b, bs_o)
    for b in range(B):
        emb = emb_buf[b * bs_e:b * bs_e + h * w * ld].view(h, w, ld)[..., :C]
        boxes = box_buf[b * bs_b:b * bs_b + n_max * 7].view(n_max, 7)
        x, y = embed_positions(boxes[:, :4], h, w)
        ref = embed_ref(emb, x, y)
        n = min(counts[b], n_max)
        got = out[b * bs_o:b * bs_o + n * C].view(n, C)
        check(got, ref[:n], embed_bound(emb, x, y, ref)[:n], f"sample_embed batched {dtype} image {b} count={counts[b]}")
        assert bool((out[b * bs_o + n * C:(b + 1) * bs_o] == -555.0).all()), f"image {b}: rows past the count were written"
    assert bool((out[B * bs_o:] == -555.0).all())


@gpu
def test_sample_embed_checks_are_not_vacuous():
    """The sampler check notices the (y0, x1) and (y1, x0) tap weights swapped."""
    g = G(3200)
    h, w, C = 13, 21, 128
    emb = torch.randn(h, w, C, generator=g).bfloat16().to(dev)
    boxes = embed_boxes(300, h, w, g).to(dev)
    out = run_sample_embed(emb, C, h, w, C, boxes, [300], 300)[:300 * C].view(300, C)
    x, y = embed_positions(boxes[:, :4], h, w)
    ref = embed_ref(emb, x, y, swap=True)
    must_fail(lambda: check(out, ref, embed_bound(emb, x, y, ref), "sample_embed vs swapped weights (must fail)"))


def test_sample_embed_reference_matches_oracle():
    """embed_ref at embed_positions equals tracker_oracle.sample_embeddings (F.grid_sample, border, align_corners=False) in float64,
    with boxes on every centre category of 2-pixel and non-square maps."""
    g = G(7)
    for h, w, C in ((2, 5, 3), (7, 2, 4), (2, 2, 1), (13, 21, 5)):
        emb = torch.randn(h, w, C, generator=g, dtype=f64)
        boxes = embed_boxes(64, h, w, g)[:, :4].double()
        x, y = embed_positions(boxes, h, w)
        want = tracker_oracle.sample_embeddings(emb.permute(2, 0, 1)[None], boxes, (h * 8, w * 8)).reshape(64, C)
        self_check(embed_ref(emb, x, y), want, f"sample_embed vs oracle h={h} w={w}")


# ================================================================================================ bi-softmax
def bisoftmax_ref(E, Mm, ld=None, lm=None, row_len=None):
    """float64 (softmax(E M^T, dim=1) + softmax(E M^T, dim=0)) / 2, zero where the labels differ.  row_len limits the row softmax
    to the first row_len columns (a wrong reference)."""
    f = E.double() @ Mm.double().t()
    fr = f if row_len is None else f[:, :row_len]
    er = torch.exp(f - fr.amax(1, keepdim=True))
    rs = er / torch.exp(fr - fr.amax(1, keepdim=True)).sum(1, keepdim=True)
    ec = torch.exp(f - f.amax(0, keepdim=True))
    cs = ec / ec.sum(0, keepdim=True)
    s = (rs + cs) / 2
    if ld is not None:
        s = torch.where(ld.double()[:, None] != lm.double()[None, :], torch.zeros_like(s), s)
    return s, rs, cs, f


def bisoftmax_bound(rs, cs, f, N, M):
    """feats are exact (grid embeddings below), so each softmax is off by: expf (2 ulps, 2^-22), f - max (|f - max| 2^-24), the sum of
    len terms (per thread len / 128 adds, a 7-level tree: (len / 128 + 8) 2^-24), the division (2^-24); plus 2^-24 for the mean."""
    kr = 4 + (M / 128 + 8) + 1 + (f - f.amax(1, keepdim=True)).abs()
    kc = 4 + (N / 128 + 8) + 1 + (f - f.amax(0, keepdim=True)).abs()
    ref = (rs + cs) / 2
    return (rs * kr + cs * kc) * U / 2 + U * ref + floor_of(ref)


def grid_embeds(n, C, g, hot=0.0):
    """Embeddings k / 8, |k| <= 12, scaled by 2 (the `hot` share of rows, whose dot products reach a few hundred and whose softmax
    saturates) or by 1/4: every product is a multiple of 2^-10 below 9 and every partial sum of 128 of them a multiple of 2^-10 below
    2^11, so E M^T is exact in fp32 in any order."""
    e = torch.randint(-12, 13, (n, C), generator=g).float() / 8
    scale = torch.where(torch.rand(n, 1, generator=g) < hot, 2.0, 0.25)
    return (e * scale).to(dev)


NM = (1, 127, 128, 129, 256, 257, 600)


@gpu
@pytest.mark.parametrize("N", NM)
@pytest.mark.parametrize("labels", [False, True])
def test_bisoftmax_edges(N, labels):
    """uc_bisoftmax with N and M around the 128-thread statistics block and the 256-wide feats blocks (the strided loops run up to
    5 times), C = 128, saturating rows; with labels every gated score must be exactly 0.  Bound: bisoftmax_bound."""
    for M in NM:
        g = G(4000 + N * 1000 + M)
        E, Mm = grid_embeds(N, 128, g, 0.3), grid_embeds(M, 128, g, 0.3)
        ld = lm = None
        if labels:
            ld = torch.randint(0, 3, (N,), generator=g).float().to(dev)
            lm = torch.randint(0, 3, (M,), generator=g).float().to(dev)
        got = ops.bisoftmax(E, Mm, ld, lm)
        ref, rs, cs, f = bisoftmax_ref(E, Mm, ld, lm)
        bound = bisoftmax_bound(rs, cs, f, N, M)
        check(got, ref, bound, f"bisoftmax N={N} M={M} labels={labels}")
        if labels:
            gate = ld[:, None] != lm[None, :]
            assert bool((got[gate] == 0).all()), "a gated score is not exactly 0"


@gpu
def test_bisoftmax_checks_are_not_vacuous():
    """The bi-softmax check notices a row statistic reduced over only the first 128 columns."""
    g = G(4100)
    E, Mm = grid_embeds(257, 128, g, 0.0), grid_embeds(600, 128, g, 0.0)
    got = ops.bisoftmax(E, Mm)
    ref, rs, cs, f = bisoftmax_ref(E, Mm, row_len=128)
    must_fail(lambda: check(got, ref, bisoftmax_bound(rs, cs, f, 257, 600), "bisoftmax vs 128-column rows (must fail)"))


def test_bisoftmax_reference_matches_definition():
    """bisoftmax_ref equals the tracker's expression (quasi_dense_embed_tracker.py:166-175) evaluated with torch.softmax in float64."""
    g = G(8)
    for N, M in ((1, 1), (129, 7), (5, 257)):
        E, Mm = torch.randn(N, 16, generator=g, dtype=f64), torch.randn(M, 16, generator=g, dtype=f64)
        f = E @ Mm.t()
        want = (f.softmax(1) + f.softmax(0)) / 2
        ld, lm = torch.randint(0, 2, (N,), generator=g).double(), torch.randint(0, 2, (M,), generator=g).double()
        self_check(bisoftmax_ref(E, Mm)[0], want, f"bisoftmax N={N} M={M}")
        gated = torch.where(ld[:, None] == lm[None, :], want, torch.zeros_like(want))
        self_check(bisoftmax_ref(E, Mm, ld, lm)[0], gated, f"bisoftmax labels N={N} M={M}")


# ================================================================================================ aligned bilinear
def ab_taps(n_out, f, n, shift=True):
    """aligned_bilinear's taps along one axis: output i samples max(i - f/2, 0) / f of the replicate-padded source (align_corners
    True): i0 = floor, i1 = min(i0 + 1, n - 1), frac.  shift=False drops the f/2 (a wrong reference)."""
    i = torch.arange(n_out, dtype=f64)
    ii = torch.clamp(i - (f // 2 if shift else 0), min=0)
    i0 = torch.floor(ii / f)
    frac = ii / f - i0
    return i0.long().clamp(max=n - 1), (i0.long() + 1).clamp(max=n - 1), frac


def ab_upsample(t, f, shift=True):
    """float64 aligned_bilinear(t, f) of t [..., h, w]: explicit four taps."""
    h, w = t.shape[-2:]
    y0, y1, fy = (a.to(t.device) for a in ab_taps(h * f, f, h, shift))
    x0, x1, fx = (a.to(t.device) for a in ab_taps(w * f, f, w, shift))
    t = t.double()
    top = t[..., y0, :][..., x0] * (1 - fx) + t[..., y0, :][..., x1] * fx
    bot = t[..., y1, :][..., x0] * (1 - fx) + t[..., y1, :][..., x1] * fx
    return top * (1 - fy)[:, None] + bot * fy[:, None]


def run_ab_add(src_buf, lds, bs_src, hs, ws, dst_buf, ldd, bs_dst, C, f, B):
    if B == 1:
        ops._lib.check(ops._L().uc_aligned_bilinear_add(ops._p(src_buf), lds, hs, ws, ops._p(dst_buf), ldd, C, f, ops._S()),
                       "uc_aligned_bilinear_add")
    else:
        ops._lib.check(ops._L().uc_aligned_bilinear_add_batched(ops._p(src_buf), lds, ctypes.c_long(bs_src), hs, ws, ops._p(dst_buf), ldd,
                                                                ctypes.c_long(bs_dst), C, f, B, ops._S()), "uc_aligned_bilinear_add_batched")
    torch.cuda.synchronize()


def ab_add_check(hs, ws, C, f, B, lds, ldd, seed, shift=True, name=""):
    """dst[..., :C] += aligned_bilinear(src[..., :C], f) on channel slices of B images with per-image padding.  The weights
    (1 - fy)(1 - fx) etc. are exact (f a power of two) and so are their products with bf16 values, so the fp32 result is the exact
    sum of 5 terms rounded up to 4 times, then once to bf16: bound 2^-8 |ref| + 4 2^-24 S (S on |terms|) + floor.  Channels outside the
    slice and the padding between images stay bitwise unchanged."""
    g = G(seed)
    bs_src, bs_dst = hs * ws * lds + (6 if B > 1 else 0), hs * f * ws * f * ldd + (10 if B > 1 else 0)
    src_buf = torch.randn(B * bs_src, generator=g).bfloat16().to(dev)
    dst_buf = torch.randn(B * bs_dst, generator=g).bfloat16().to(dev)
    before = dst_buf.clone()
    run_ab_add(src_buf, lds, bs_src, hs, ws, dst_buf, ldd, bs_dst, C, f, B)
    inside = torch.zeros(B * bs_dst, dtype=torch.bool, device=dev)
    worst = 0.0
    for b in range(B):
        src = src_buf[b * bs_src:b * bs_src + hs * ws * lds].view(hs, ws, lds)[..., :C].permute(2, 0, 1)
        d0 = before[b * bs_dst:b * bs_dst + hs * f * ws * f * ldd].view(hs * f, ws * f, ldd)[..., :C].permute(2, 0, 1).double()
        got = dst_buf[b * bs_dst:b * bs_dst + hs * f * ws * f * ldd].view(hs * f, ws * f, ldd)[..., :C].permute(2, 0, 1)
        up = ab_upsample(src, f, shift)
        ref = d0 + up
        S = d0.abs() + ab_upsample(src.abs(), f, shift)
        worst = max(worst, check(got, ref, REL * ref.abs() + 4 * U * S + floor_of(ref),
                                 f"aligned_bilinear_add {name} hs={hs} ws={ws} C={C} f={f} B={B} lds={lds} ldd={ldd} image {b}"))
        inside[b * bs_dst:b * bs_dst + hs * f * ws * f * ldd].view(hs * f, ws * f, ldd)[..., :C] = True
    assert torch.equal(dst_buf[~inside], before[~inside]), "aligned_bilinear_add wrote outside its channel slice / images"
    return worst


@gpu
@pytest.mark.parametrize("f", [1, 2, 4, 8])
@pytest.mark.parametrize("C", [2, 8, 130])
def test_aligned_bilinear_add_edges(f, C):
    """uc_aligned_bilinear_add (B = 1) and _batched (B = 3, padded per-image strides) with hs or ws = 1, odd sizes, and lds / ldd > C
    (channel slices of wider maps).  Bound: ab_add_check."""
    for i, (hs, ws) in enumerate([(1, 1), (1, 7), (5, 1), (3, 5), (9, 4)]):
        ab_add_check(hs, ws, C, f, 1, C + 6, C + 4, 5000 + i)
        ab_add_check(hs, ws, C, f, 3, C + 2, C + 8, 5100 + i)


@gpu
@pytest.mark.parametrize("hs,ws,f", [(20, 20, 2), (10, 10, 4), (50, 80, 2), (25, 40, 4)])
def test_aligned_bilinear_add_production(hs, ws, f):
    """The mask branch's fusions of P4 (f = 2) and P5 (f = 4) into P3 at 320x320 and 800x1280 inputs, C = 128, B = 1 and 2."""
    ab_add_check(hs, ws, 128, f, 1, 128, 128, 5200 + hs)
    ab_add_check(hs, ws, 128, f, 2, 128, 128, 5300 + hs)


@gpu
def test_aligned_bilinear_add_checks_are_not_vacuous():
    """The check notices the f/2 shift of aligned_bilinear dropped."""
    must_fail(lambda: ab_add_check(9, 4, 8, 4, 1, 8, 8, 5004, shift=False, name="(vs no f/2 shift, must fail)"))


def test_aligned_bilinear_reference_matches_oracle():
    """ab_upsample equals unicorn_oracle.aligned_bilinear (replicate pad, interpolate align_corners=True, pad f/2, crop) in float64."""
    g = G(9)
    for hs, ws in ((1, 1), (1, 7), (5, 1), (3, 5)):
        t = torch.randn(2, 3, hs, ws, generator=g, dtype=f64)
        for f in (1, 2, 4, 8):
            self_check(ab_upsample(t, f), orc.aligned_bilinear(t, f), f"aligned_bilinear hs={hs} ws={ws} f={f}")


# ================================================================================================ CondInst mask head
STRIDES = (8, 16, 32)
SOI = (64.0, 128.0, 256.0)


def mask_instances(dyn, level_hw, anchors):
    """Per instance: its 169 parameters, location ((ai % w) + 0.5) * stride, ((ai / w) + 0.5) * stride and soi, from the anchor index
    into the levels' concatenation (dyn: 3 tensors [hk, wk, ld_dyn])."""
    starts = [0, level_hw[0][0] * level_hw[0][1], level_hw[0][0] * level_hw[0][1] + level_hw[1][0] * level_hw[1][1]]
    prm, loc, soi, lvl = [], [], [], []
    for a in anchors:
        k = 2 if a >= starts[2] else (1 if a >= starts[1] else 0)
        ai = a - starts[k]
        w = level_hw[k][1]
        prm.append(dyn[k].reshape(-1, dyn[k].shape[-1])[ai, :169])
        loc.append([((ai % w) + 0.5) * STRIDES[k], ((ai // w) + 0.5) * STRIDES[k]])
        soi.append(SOI[k])
        lvl.append(k)
    dv = dyn[0].device
    return (torch.stack(prm).double() if prm else torch.zeros(0, 169, dtype=f64, device=dv)), torch.tensor(loc, dtype=f64, device=dv).reshape(-1, 2), \
        torch.tensor(soi, dtype=f64, device=dv), torch.tensor(lvl, device=dv)


def mask_logits(feats, prm, loc, soi, center=4, absolute=False):
    """float64 instance logits [n, h, w]: rel = (loc - (8 px + center)) / soi, then three explicit 1x1 layers 10 -> 8 -> 8 -> 1
    (weights 80 | 64 | 8, biases 8 | 8 | 1) with ReLU.  absolute=True: every operand by its absolute value and ReLU by the identity
    (the sum of |terms| of each output).  center=0 drops the + stride / 2 of compute_locations (a wrong reference)."""
    h, w = feats.shape[:2]
    n = prm.shape[0]
    px = torch.arange(w, dtype=f64, device=feats.device) * 8 + center
    py = torch.arange(h, dtype=f64, device=feats.device) * 8 + center
    rx = (loc[:, 0, None, None] - px[None, None, :]) / soi[:, None, None]
    ry = (loc[:, 1, None, None] - py[None, :, None]) / soi[:, None, None]
    x = torch.cat([rx.expand(n, h, w)[:, None], ry.expand(n, h, w)[:, None],
                   feats.double().permute(2, 0, 1)[None].expand(n, -1, -1, -1)], 1)  # [n, 10, h, w]
    p = prm.abs() if absolute else prm
    act = (lambda t: t) if absolute else F.relu
    if absolute:
        x = x.abs()
    w0, w1, w2 = p[:, :80].reshape(n, 8, 10), p[:, 80:144].reshape(n, 8, 8), p[:, 144:152].reshape(n, 1, 8)
    b0, b1, b2 = p[:, 152:160], p[:, 160:168], p[:, 168:169]
    x = act(torch.einsum("noi,nihw->nohw", w0, x) + b0[:, :, None, None])
    x = act(torch.einsum("noi,nihw->nohw", w1, x) + b1[:, :, None, None])
    return (torch.einsum("noi,nihw->nohw", w2, x) + b2[:, :, None, None])[:, 0]


def convex_up(v, um, up, last_row_pad=False):
    """float64 convex upsampling of v [n, h, w] by up with the 9-way softmax weights of um [h, w, 9 up up] (channel k up^2 + i up + j,
    neighbour k = (dy + 1) * 3 + dx + 1, zero padding) -> ([n, h up, w up], the softmax [h, w, 9, up, up]).  last_row_pad=True also
    zeroes the last row's taps (a wrong reference)."""
    n, h, w = v.shape
    p = torch.softmax(um.double().reshape(h, w, 9, up, up), 2)
    pad = F.pad(v.double(), (1, 1, 1, 1))
    if last_row_pad:
        pad[:, h] = 0
    nb = torch.stack([pad[:, dy:dy + h, dx:dx + w] for dy in range(3) for dx in range(3)], 1)  # [n, 9, h, w]
    out = torch.einsum("yxkij,nkyx->nyixj", p, nb).reshape(n, h * up, w * up)
    return out, p


def mask_reference(feats, um, dyn, level_hw, anchors, up, d, center=4, last_row_pad=False):
    """float64 masks of the instances at `anchors` [n, h up d, w up d] and the bound.
    Bound, stage by stage (first order; a factor 2 on the propagated terms absorbs the rest):
      logits: three layers of 11, 9, 9 terms, each product and add rounded (2 per term), and each layer's input error passed through
              its weights: e_logit <= 60 2^-24 A, A = mask_logits(absolute=True);
      convex: acc = sum_k p_k v_k with p_k off by expf (2 ulps), x - max (|x - max| ulps), the 9-term denominator (8 + 4), the division
              and the product, and 9 adds: e_acc <= (27 + max|x - max|) 2^-24 sum p_k |v_k| + sum p_k e_logit_k;
      sigmoid: 1 / (1 + expf(-acc)) within 6 2^-24 relative, and sigma (1 - sigma) e_acc from acc;
      final:  aligned_bilinear x d has exact weights (d a power of two): sum w e_sigma + 6 2^-24 sum w sigma."""
    prm, loc, soi, _ = mask_instances(dyn, level_hw, anchors)
    lg = mask_logits(feats, prm, loc, soi, center)
    A = mask_logits(feats, prm, loc, soi, center, absolute=True)
    acc, p = convex_up(lg, um, up, last_row_pad)
    h, w = lg.shape[1:]
    xm = um.double().reshape(h, w, 9, up, up)
    spread = (xm - xm.amax(2, keepdim=True)).abs().amax(2)  # [h, w, up, up]
    spread = spread.permute(0, 2, 1, 3).reshape(h * up, w * up)
    av, _ = convex_up(lg.abs(), um, up)
    ae, _ = convex_up(60 * U * A, um, up)
    e_acc = (27 + spread) * U * av + ae
    sig = torch.sigmoid(acc)
    e_sig = 6 * U * sig + 2 * sig * (1 - sig) * e_acc
    if d == 1:
        return sig, e_sig + floor_of(sig)
    ref = ab_upsample(sig, d)
    return ref, ab_upsample(e_sig, d) + 6 * U * ref + floor_of(ref)


def mask_case(h, w, level_hw, up, ld_dyn, g, B=1, S=1, pad=(0, 0, 0)):
    """Mask-branch and controller inputs: feats [S, h, w, 8]; up_masks [S, h, w, 9 up^2] with random pixels, pixels whose 9 weights
    tie and pixels where one weight dominates by 120 (saturated); controller outputs [B, hk, wk, ld_dyn] as views of buffers with
    `pad` extra elements per image (bs_dyn > hk wk ld_dyn), with biases drawn so hidden pre-activations fall near zero, and every
    third anchor's last bias at +-30 (saturated sigmoid)."""
    feats = torch.randn(S, h, w, 8, generator=g)
    um = torch.randn(S, h, w, 9, up * up, generator=g) * 3
    kind = torch.randint(0, 3, (S, h, w, 1, 1), generator=g)
    um = torch.where(kind == 1, torch.full_like(um, 0.75), um)
    big = torch.full_like(um, -60.0)
    big.scatter_(3, torch.randint(0, 9, (S, h, w, 1, up * up), generator=g), 60.0)
    um = torch.where(kind == 2, big, um)
    dyn = []
    for k, (hk, wk) in enumerate(level_hw):
        bs = hk * wk * ld_dyn + pad[k]
        buf = torch.randn(B * bs, generator=g) * 0.5
        v = buf.as_strided((B, hk, wk, ld_dyn), (bs, wk * ld_dyn, ld_dyn, 1))
        v[..., 152:168] *= 0.1
        v[:, :, :, 168] = torch.where(torch.rand(B, hk, wk, generator=g) < 0.33, torch.sign(torch.randn(B, hk, wk, generator=g)) * 30.0,
                                      v[:, :, :, 168])
        v[..., 169:] = float("nan")  # the padding columns of a ld_dyn row are never read
        dyn.append(buf.to(dev).as_strided((B, hk, wk, ld_dyn), (bs, wk * ld_dyn, ld_dyn, 1)))
    return feats.to(dev), um.reshape(S, h, w, 9 * up * up).to(dev), dyn


def edge_anchors(level_hw, g, n):
    """Anchors on purpose: the first and last anchor of each level (start[k], start[k+1] - 1), the first and last column of a middle
    row, then random ones, n in all."""
    a, s = [], 0
    for hk, wk in level_hw:
        r = hk // 2
        a += [s, s + hk * wk - 1, s + r * wk, s + r * wk + wk - 1]
        s += hk * wk
    while len(a) < n:
        a.append(int(torch.randint(0, s, (1,), generator=g)))
    return a[:n]


MASK_MAPS = [((5, 7), [(5, 7), (3, 4), (2, 2)]), ((13, 21), [(13, 21), (7, 11), (4, 6)])]


@gpu
@pytest.mark.parametrize("up,d", [(1, 1), (4, 2), (8, 1), (2, 4)])
@pytest.mark.parametrize("ld_dyn", [169, 176])
def test_dynamic_masks_edges(up, d, ld_dyn):
    """uc_dynamic_masks with anchors chosen on purpose (ws.anchors / ws.count filled directly), maps with h w < 256 and not a multiple
    of 256, the production rates (4, 2) and (8, 1) and the edges (1, 1) and (2, 4), ld_dyn 169 and 176, count 0, 1 and > n_max:
    rows past min(count, n_max) keep their sentinel.  Bound: mask_reference."""
    for mi, ((h, w), level_hw) in enumerate(MASK_MAPS):
        g = G(6000 + 10 * up + d + mi + ld_dyn)
        feats, um, dyn = mask_case(h, w, level_hw, up, ld_dyn, g)
        A = sum(a * b for a, b in level_hw)
        n_max = 16
        anchors = edge_anchors(level_hw, g, n_max)
        ref, bound = mask_reference(feats[0], um[0], [t[0] for t in dyn], level_hw, anchors, up, d)
        ws = ops.PostWorkspace(A, dev)
        ws.anchors[:n_max] = torch.tensor(anchors, dtype=torch.int32, device=dev)
        for count in (0, 1, n_max + 5):
            ws.count.fill_(count)
            H, W = h * up * d, w * up * d
            out = torch.full((n_max, H, W), -5.0, device=dev)
            ops.dynamic_masks(feats, um, dyn, level_hw, ws, n_max, up_rate=up, d_rate=d, out=out)
            torch.cuda.synchronize()
            n = min(count, n_max)
            check(out[:n], ref[:n], bound[:n], f"dynamic_masks h={h} w={w} up={up} d={d} ld={ld_dyn} count={count}")
            assert bool((out[n:] == -5.0).all()), "rows past the count were written"


@gpu
def test_dynamic_masks_batched_edges():
    """uc_dynamic_masks_batched: B = 4 head images over S = 2 mask-branch images, image_of = [1, -1, 0, 2] (the -1 and S entries are
    skipped and their output slabs stay untouched), controller outputs with per-image strides larger than hk wk ld_dyn and distinct
    per level, distinct counts; each image against its own reference."""
    g = G(6500)
    (h, w), level_hw = MASK_MAPS[1]
    up, d, ld_dyn, B, S, n_max = 4, 2, 176, 4, 2, 9
    feats, um, dyn = mask_case(h, w, level_hw, up, ld_dyn, g, B=B, S=S, pad=(8, 40, 2))
    A = sum(a * b for a, b in level_hw)
    ws = ops.PostWorkspace(A, dev, batch=B)
    anchors = [edge_anchors(level_hw, g, n_max + 3)[::-1][:n_max] for _ in range(B)]
    for b in range(B):
        ws.anchors[b, :n_max] = torch.tensor(anchors[b], dtype=torch.int32, device=dev)
    counts = [5, 3, n_max + 2, 1]
    ws.count.copy_(torch.tensor(counts, dtype=torch.int32))
    image_of = torch.tensor([1, -1, 0, S], dtype=torch.int32, device=dev)
    out = torch.full((B, n_max, h * up * d, w * up * d), -5.0, device=dev)
    ops.dynamic_masks(feats, um, dyn, level_hw, ws, n_max, up_rate=up, d_rate=d, out=out, image_of=image_of)
    torch.cuda.synchronize()
    for b in range(B):
        img = int(image_of[b])
        if not 0 <= img < S:
            assert bool((out[b] == -5.0).all()), f"skipped head image {b} (image_of {img}) was written"
            continue
        n = min(counts[b], n_max)
        ref, bound = mask_reference(feats[img], um[img], [t[b] for t in dyn], level_hw, anchors[b][:n], up, d)
        check(out[b, :n], ref, bound, f"dynamic_masks batched image {b} (mask image {img}) count={counts[b]}")
        assert bool((out[b, n:] == -5.0).all())


@gpu
def test_dynamic_masks_checks_are_not_vacuous():
    """The mask check notices the + stride / 2 of compute_locations dropped and the convex upsample's last row treated as padding."""
    g = G(6000 + 10 * 4 + 2 + 1 + 169)
    (h, w), level_hw = MASK_MAPS[1]
    feats, um, dyn = mask_case(h, w, level_hw, 4, 169, g)
    n_max = 16
    anchors = edge_anchors(level_hw, g, n_max)
    ws = ops.PostWorkspace(sum(a * b for a, b in level_hw), dev)
    ws.anchors[:n_max] = torch.tensor(anchors, dtype=torch.int32, device=dev)
    ws.count.fill_(n_max)
    out = ops.dynamic_masks(feats, um, dyn, level_hw, ws, n_max, up_rate=4, d_rate=2)
    for kw, what in ((dict(center=0), "no + 4"), (dict(last_row_pad=True), "last row as padding")):
        ref, bound = mask_reference(feats[0], um[0], [t[0] for t in dyn], level_hw, anchors, 4, 2, **kw)
        must_fail(lambda: check(out, ref, bound, f"dynamic_masks vs {what} (must fail)"))


def test_mask_reference_matches_oracle():
    """mask_logits + convex_up + sigmoid (+ ab_upsample x d) equal unicorn_oracle.dynamic_masks followed by aligned_bilinear x d_rate
    in float64, for edge anchors of every level, at every (up, d) tested on the GPU."""
    g = G(10)
    (h, w), level_hw = MASK_MAPS[0]
    for up, d in ((1, 1), (4, 2), (8, 1), (2, 4)):
        feats = torch.randn(h, w, 8, generator=g, dtype=f64)
        um = torch.randn(h, w, 9 * up * up, generator=g, dtype=f64) * 3
        dyn = [torch.randn(hk, wk, 176, generator=g, dtype=f64) * 0.5 for hk, wk in level_hw]
        anchors = edge_anchors(level_hw, g, 14)
        prm, loc, soi, lvl = mask_instances(dyn, level_hw, anchors)
        mine = torch.sigmoid(convex_up(mask_logits(feats, prm, loc, soi), um, up)[0])
        if d > 1:
            mine = ab_upsample(mine, d)
        want = orc.dynamic_masks(feats.permute(2, 0, 1)[None], prm, loc, lvl, um.permute(2, 0, 1)[None], up_rate=up, soi=SOI)
        self_check(mine, orc.aligned_bilinear(want, d)[:, 0], f"mask head up={up} d={d}")


# ================================================================================================ bilinear resize
def resize_src(n_out, n_in, scale, dtype):
    """PyTorch's source coordinate (upsample_bilinear2d, align_corners=False) of every output index, in `dtype`: max((i + 0.5) *
    scale - 0.5, 0), scale = 1 / scale_factor when given, else n_in / n_out."""
    sc = torch.tensor(scale if scale > 0 else n_in, dtype=dtype)
    if scale <= 0:
        sc = sc / torch.tensor(n_out, dtype=dtype)
    i = torch.arange(n_out, dtype=dtype)
    return torch.clamp((i + 0.5) * sc - 0.5, min=0)


def resize_ref(src, fy, fx, half_shift=False):
    """float64 bilinear resize of src [P, Hs, Ws] at source coordinates fy [Hd], fx [Wd]: i0 = min(floor(f), n - 1), i1 = min(i0 + 1,
    n - 1), lambda = clamp(f - i0, 0, 1) (guard_index_and_lambda).  half_shift=True samples half a pixel further (a wrong reference)."""
    Hs, Ws = src.shape[-2:]

    def taps(f, n):
        f = f.double().to(src.device) + (0.5 if half_shift else 0.0)
        i0 = torch.floor(f).long().clamp(max=n - 1)
        return i0, (i0 + 1).clamp(max=n - 1), (f - i0).clamp(0, 1)
    y0, y1, ly = taps(fy, Hs)
    x0, x1, lx = taps(fx, Ws)
    s = src.double()
    top = s[:, y0][:, :, x0] * (1 - lx) + s[:, y0][:, :, x1] * lx
    bot = s[:, y1][:, :, x0] * (1 - lx) + s[:, y1][:, :, x1] * lx
    return top * (1 - ly)[:, None] + bot * ly[:, None]


def resize_bound(src, fy, fx, ref):
    """fp32: 1 - l, two products and a sum per row, the outer products and sum: 6 2^-24 S (S on |v|); position term with 2 ulps of
    (|fy| + |fx| + 2) x 2 max|v| of the plane (the kernel may contract (i + 0.5) * scale - 0.5)."""
    S = resize_ref(src.abs(), fy, fx)
    vmax = src.double().abs().amax((1, 2))[:, None, None]
    X = 2 * U * (fy.double().to(src.device)[:, None] + fx.double().to(src.device)[None, :] + 2) * 2 * vmax
    return 6 * U * S + X + floor_of(ref)


BILINEAR_CASES = [(3, 64, 48, 32, 24, 2.0), (2, 64, 64, 16, 16, 4.0), (1, 320, 320, 40, 40, 8.0), (4, 7, 7, 3, 3, 0.0),
                  (2, 7, 10, 3, 4, 0.0), (3, 3, 3, 50, 50, 0.0), (2, 1, 9, 4, 5, 0.0), (2, 6, 1, 13, 2, 0.0), (2, 1, 1, 3, 4, 0.0),
                  (48, 25, 40, 100, 160, 0.0)]


@gpu
@pytest.mark.parametrize("P,Hs,Ws,Hd,Wd,sc", BILINEAR_CASES)
def test_bilinear_edges(P, Hs, Ws, Hd, Wd, sc):
    """uc_bilinear_f32: downscaling by scale factors 2, 4, 8 and by size ratios such as 7 -> 3, upscaling 3 -> 50, Hs or Ws = 1, and
    P Hd Wd > num_sms * 16 * 256 (the grid-stride loop runs several times).  Positions in fp32 as PyTorch computes them; bound
    resize_bound."""
    g = G(7000 + Hs * Ws + Hd)
    src = torch.randn(P, Hs, Ws, generator=g).to(dev)
    if P == 48:
        assert P * Hd * Wd > num_sms() * 16 * 256
    out = ops.bilinear(src, Hd, Wd, sc, sc)
    fy, fx = resize_src(Hd, Hs, sc, torch.float32), resize_src(Wd, Ws, sc, torch.float32)
    ref = resize_ref(src, fy, fx)
    check(out, ref, resize_bound(src, fy, fx, ref), f"bilinear P={P} {Hs}x{Ws} -> {Hd}x{Wd} scale={sc}")


@gpu
def test_bilinear_checks_are_not_vacuous():
    """The resize check notices a half-pixel shift of the source coordinate."""
    g = G(7100)
    src = torch.randn(3, 7, 10, generator=g).to(dev)
    out = ops.bilinear(src, 3, 4)
    fy, fx = resize_src(3, 7, 0.0, torch.float32), resize_src(4, 10, 0.0, torch.float32)
    ref = resize_ref(src, fy, fx, half_shift=True)
    must_fail(lambda: check(out, ref, resize_bound(src, fy, fx, ref), "bilinear vs half-pixel shift (must fail)"))


def test_bilinear_reference_matches_interpolate():
    """resize_ref at float64 source coordinates equals F.interpolate(bilinear, align_corners=False) in float64, by size and by scale
    factor, down and up, with 1-pixel sides."""
    g = G(11)
    for P, Hs, Ws, Hd, Wd, sc in BILINEAR_CASES[:-1]:
        src = torch.randn(P, Hs, Ws, generator=g, dtype=f64)
        if sc > 0:
            want = F.interpolate(src[None], scale_factor=1 / sc, mode="bilinear", align_corners=False)[0]
        else:
            want = F.interpolate(src[None], size=(Hd, Wd), mode="bilinear", align_corners=False)[0]
        got = resize_ref(src, resize_src(Hd, Hs, sc, f64), resize_src(Wd, Ws, sc, f64))
        self_check(got, want, f"bilinear {Hs}x{Ws} -> {Hd}x{Wd} scale={sc}")

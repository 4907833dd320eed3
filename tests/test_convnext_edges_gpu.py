"""Edge-case parity of the ConvNeXt block kernels against float64 references on the same rounded operands: the depthwise 7x7
(uc_dwconv7 with fp32 taps and its LayerNorm statistics, uc_dwconv7_mma with bf16 taps), the fused MLP back half
(uc_convnext_mlp), the depthwise 7x7 + LayerNorm (uc_dwconv7_ln, every dispatch target) and the LayerNorm folded into pwconv1
(uc_dwconv7 ln_stats -> uc_conv2d row_stats).  Shapes sit on tile seams, partial tiles, partial channel chunks, maps smaller than
the window, row counts around the 128-row tile and multi-pass persistent schedules.

Bounds are per element: |got - ref| <= 2^-8 |ref| (one rounding of the output to bf16, whose unit roundoff is 2^-8) + an
accumulation term derived in each reference's docstring + a small floor.  Every check prints its largest
err / bound, and the checks that could pass by accident are run once against a wrong reference, where they must fail."""
import math

import pytest
import torch
import torch.nn.functional as F

from unicorn_b200 import ops

pytestmark = pytest.mark.gpu
dev = "cuda"
REL = 2.0 ** -8  # one rounding to bf16 (8 significant bits, round to nearest)
U = 2.0 ** -24   # fp32 unit roundoff
FIX = 2.0 ** 22  # fixed-point scale of the LayerNorm statistics (kGnFixedScale)
GELU_FIT = 4e-6  # |GELU fit - erf GELU| over the real line (test_gelu_fit.py)
GELU_DMAX = 1.13  # max |GELU'(z)| = 1.1289 at z = sqrt(2)
EDGE_HW = [(1, 1), (1, 9), (3, 2), (7, 7), (8, 17), (9, 16), (15, 33), (16, 8), (17, 31), (31, 15), (33, 9), (33, 33)]
SEAMS = (8, 9, 15, 16, 17, 31, 33)  # around the 16 x 8 (TMA) and 16 x 16 (MMA) output tiles
EDGE_C = (8, 24, 40, 72, 104, 200)  # partial 32-channel (MMA) and 64-channel (TMA) chunks


def G(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def check(got, ref, bound, name):
    """Per-element |got - ref| <= bound; ref and bound float64."""
    err = (got.double() - ref).abs()
    ratio = (err / bound).max().item()
    print(f"err/bound {ratio:.3f}  {name}")
    assert ratio <= 1.0, f"{name}: max err/bound {ratio:.3g} (max err {err.max().item():.3g})"
    return ratio


def ulp_bf16(v):
    """Spacing of the bf16 numbers at |v| (0 at v = 0)."""
    _, e = torch.frexp(v)
    return torch.where(v == 0, torch.zeros_like(v), torch.ldexp(torch.ones_like(v), e - 8))


def offset_values(n, base, ratio, g):
    """n bf16 values with mean ~base and std ~|base| / ratio, all exactly representable: base + k * ulp(base) (as in
    test_kernel_edges_gpu).  When the std is below one ulp, a fraction of the values sits one ulp off base."""
    ulp = 2.0 ** (math.floor(math.log2(abs(base))) - 7)
    sigma = abs(base) / ratio
    if sigma >= ulp:
        k = torch.round(torch.randn(n, generator=g, dtype=torch.float64) * sigma / ulp)
    else:
        p = (sigma / ulp) ** 2
        u = torch.rand(n, generator=g, dtype=torch.float64)
        k = (u < p / 2).double() - ((u >= p / 2) & (u < p)).double()
    return base + k * ulp


def nchw(t):
    return t.permute(0, 3, 1, 2)


def nhwc(t):
    return t.permute(0, 2, 3, 1)


# ---------------------------------------------------------------------------------------------------------------- depthwise 7x7
def dw_mma_taps(q, C):
    """The bf16 taps [C,1,7,7] and fp32 biases [C] that the operand of uc_dwconv7_mma carries (ops.pack_dw_weight_mma: per
    32-channel chunk [32][7][8] tap pairs {e[j-1], e[j]} with e[-1] = 0, then 32 biases): tap k is the low half of pair k + 1."""
    nch = q.shape[0]
    lo = q[:, :1792].reshape(nch, 32, 7, 8)[..., 1:8] & 0xFFFF
    taps = ((lo ^ 0x8000) - 0x8000).to(torch.int16).view(torch.bfloat16).double()
    bias = q[:, 1792:].contiguous().view(torch.float32).reshape(-1)
    return taps.reshape(nch * 32, 1, 7, 7)[:C], bias[:C].double()


def run_tma(x, w, b, **kw):
    return ops.dwconv7(x, ops.pack_dw_weight(w), b, **kw)


def run_mma(x, w, b, **kw):
    kw.pop("ln_stats", None)
    return ops.dwconv7_mma(x, ops.pack_dw_weight_mma(w, b), **kw)


KERNELS = {"tma": run_tma, "mma": run_mma}


def lattice_taps(C):
    """Taps (64 + (37 k + 11 c) mod 192) / 64 * +-2^{-1,0,1}: exact in bf16, none zero, the 49 taps of a channel all different and
    neighbouring channels different sets, so an output names the (channel, tap) it came from."""
    c = torch.arange(C, dtype=torch.float64)[:, None]
    k = torch.arange(49, dtype=torch.float64)[None]
    n = 64 + torch.remainder(37 * k + 11 * c, 192)
    s = torch.where(c % 2 == 0, 1.0, -1.0) * 2.0 ** (torch.div(c, 2, rounding_mode="floor") % 3 - 1)
    return (n / 64 * s).reshape(C, 1, 7, 7)


@pytest.mark.parametrize("C", EDGE_C)
def test_dwconv7_impulse_lattice_bitwise(C):
    """Zero bias and a map that is 0 except 1.0 at every pixel (7 i + oy, 7 j + ox): every 7x7 window holds exactly one impulse,
    or none near a border, so every output is exactly one tap (or 0) and both kernels must match the float64 convolution bit for
    bit.  Image b of the batch uses phase b (all 49 phases in one launch, so a tap read from the wrong image shows), on maps
    smaller than the window, on every combination of H, W around the tile seams, and on partial channel chunks."""
    w = lattice_taps(C)
    wd = w.to(dev)
    wf = w.float().to(dev)
    b = torch.zeros(C, device=dev)
    phases = [(oy, ox) for oy in range(7) for ox in range(7)]
    shapes = EDGE_HW[:4] + [(h, w_) for h in SEAMS for w_ in SEAMS]
    hit = 0
    for H, W in shapes:
        xb = torch.zeros(len(phases), H, W, C, dtype=torch.bfloat16, device=dev)
        for i, (oy, ox) in enumerate(phases):
            xb[i, oy::7, ox::7, :] = 1.0
        want = nhwc(F.conv2d(nchw(xb.double()), wd, padding=3, groups=C)).bfloat16()
        hit += int((want != 0).sum().item())
        for name, run in KERNELS.items():
            got = run(xb, wf, b)
            if not torch.equal(got, want):
                bad = (got != want).nonzero()
                raise AssertionError(f"dwconv7 {name} impulse lattice C={C} H={H} W={W}: {bad.shape[0]} wrong outputs, first "
                                     f"(phase, h, w, c) = {[phases[bad[0, 0]]] + bad[0, 1:].tolist()}: got {got[tuple(bad[0])].item()}"
                                     f" want {want[tuple(bad[0])].item()}")
    assert hit > 0
    print(f"impulse lattice C={C}: {len(shapes)} maps x 49 phases, {hit} non-zero outputs, both kernels bitwise")


def dw_ref(x, w, b):
    """float64 depthwise convolution of the stored bf16 map and S = |b| + sum |x| |w|, which bounds every partial sum."""
    C = x.shape[3]
    xd = nchw(x.double())
    ref = nhwc(F.conv2d(xd, w.double(), b.double(), padding=3, groups=C))
    S = nhwc(F.conv2d(xd.abs(), w.double().abs(), b.double().abs(), padding=3, groups=C))
    return ref, S


# fp32 accumulation: the TMA kernel starts from the bias and adds 49 products with one FMA rounding (<= u * |partial sum| <= u * S)
# each; the MMA kernel runs 7 mma.sync of K = 16 per output, each of which may round twice (the products are exact in fp32) and
# truncate rather than round (2 u): 7 * 2 * 2 = 28
DW_C = {"tma": 49, "mma": 28}
DW_FLOOR = 1e-7


def dw_bound(ref, S, kernel):
    return ref.abs() * REL + DW_C[kernel] * U * S + DW_FLOOR


def dw_case(C, H, W, B, seed):
    g = G(seed)
    x = torch.randn(B, H, W, C, generator=g).to(dev).bfloat16()
    w = (torch.randn(C, 1, 7, 7, generator=g) / 7).to(dev)
    b = torch.randn(C, generator=g).to(dev)
    return x, w, b


DW_PROD = [(96, 20, 28), (192, 17, 23), (256, 10, 16), (1536, 5, 9), (384, 33, 40), (768, 50, 80), (192, 200, 320),
           (1536, 25, 40), (256, 100, 160), (104, 9, 3)]


@pytest.mark.parametrize("C,H,W,B", [(C, H, W, 2) for C, H, W in DW_PROD] + [(C, 0, 0, 3) for C in EDGE_C])
def test_dwconv7_random_per_element(C, H, W, B):
    """Random maps against float64: uc_dwconv7 against the fp32 taps, uc_dwconv7_mma against the bf16 taps its operand carries
    (decoded from the operand itself).  H = W = 0 stands for every edge map of EDGE_HW at this channel count."""
    shapes = EDGE_HW if H == 0 else [(H, W)]
    for i, (h, w_) in enumerate(shapes):
        x, w, b = dw_case(C, h, w_, B, 100 + C + i)
        ref, S = dw_ref(x, w, b)
        check(run_tma(x, w, b), ref, dw_bound(ref, S, "tma"), f"dwconv7 tma C={C} H={h} W={w_} B={B}")
        wq, bq = dw_mma_taps(ops.pack_dw_weight_mma(w, b), C)
        refq, Sq = dw_ref(x, wq, bq)
        check(run_mma(x, w, b), refq, dw_bound(refq, Sq, "mma"), f"dwconv7 mma C={C} H={h} W={w_} B={B}")


def test_dwconv7_checks_are_not_vacuous():
    """The per-element bound tells the tap precisions apart: the fp32-tap kernel fails against the bf16-tap reference and the
    bf16-tap kernel against the fp32-tap one (small outputs carry tap-rounding errors far above the accumulation term)."""
    x, w, b = dw_case(96, 20, 28, 2, 7)
    ref, S = dw_ref(x, w, b)
    wq, bq = dw_mma_taps(ops.pack_dw_weight_mma(w, b), 96)
    refq, Sq = dw_ref(x, wq, bq)
    with pytest.raises(AssertionError):
        check(run_tma(x, w, b), refq, dw_bound(refq, Sq, "tma"), "dwconv7 tma vs bf16 taps (must fail)")
    with pytest.raises(AssertionError):
        check(run_mma(x, w, b), ref, dw_bound(ref, S, "mma"), "dwconv7 mma vs fp32 taps (must fail)")


@pytest.mark.parametrize("kernel", ["tma", "mma"])
@pytest.mark.parametrize("C", EDGE_C)
def test_dwconv7_batch_schedule_and_guards(kernel, C):
    """Image b of a B = 3 launch is bitwise the B = 1 launch of that image; the atomic-counter schedule gives the bits of the
    static one; the output is the first 3 images of a 4-image buffer whose last image (the guard) and the input stay unchanged."""
    run = KERNELS[kernel]
    for i, (H, W) in enumerate(EDGE_HW):
        x, w, b = dw_case(C, H, W, 3, 200 + C + i)
        x0 = x.clone()
        buf = torch.randn(4, H, W, C, generator=G(i)).to(dev).bfloat16()
        buf0 = buf.clone()
        out = run(x, w, b, out=buf[:3])
        tag = f"dwconv7 {kernel} C={C} H={H} W={W}"
        assert torch.equal(buf[3], buf0[3]), f"{tag}: guard image overwritten"
        assert torch.equal(x, x0), f"{tag}: input changed"
        for k in range(3):
            assert torch.equal(out[k], run(x[k:k + 1].contiguous(), w, b)[0]), f"{tag}: image {k} differs from its B = 1 launch"
        ctr = torch.zeros(1, dtype=torch.int32, device=dev)
        assert torch.equal(out, run(x, w, b, work_counter=ctr)), f"{tag}: counter schedule differs from the static one"


@pytest.mark.parametrize("C,H,W", [(C, H, W) for C in EDGE_C for H, W in ((7, 7), (17, 31), (33, 9))] + [(768, 50, 80), (1536, 5, 9)])
def test_dwconv7_ln_stats(C, H, W):
    """The per-pixel {sum, sum of squares} over C of the stored bf16 outputs, fixed point 2^22, are ADDED to the buffer (pre-filled
    here).  Per 64-channel chunk the kernel sums in fp32 (a tree of depth 6 over the 64 values: <= 6 u sum|y|, fma for the
    squares: 7 u) and rounds once to the fixed point (<= 2^-23 each), so |st / 2^22 - sum y| <= n_chunks 2^-22 + 2^-19 sum |y|
    (and the same for sum y^2, with 2^-19 > 7 u).  A B = 3 launch gives each image the statistics of its B = 1 launch."""
    B = 3
    x, w, b = dw_case(C, H, W, B, 300 + C + H)
    pre = torch.randint(-2 ** 40, 2 ** 40, (B * H * W, 2), generator=G(C), dtype=torch.int64).to(dev)
    st = pre.clone()
    out = run_tma(x, w, b, ln_stats=st)
    nch = -(-C // 64)
    y = out.double().reshape(-1, C)
    got = (st - pre).double() / FIX
    for j, (want, mag) in enumerate(((y.sum(1), y.abs().sum(1)), ((y * y).sum(1), (y * y).sum(1)))):
        check(got[:, j], want, nch * 2.0 ** -22 + 2.0 ** -19 * mag, f"ln_stats {'sum' if j == 0 else 'sumsq'} C={C} H={H} W={W}")
    for k in range(B):
        st1 = torch.zeros(H * W, 2, dtype=torch.int64, device=dev)
        run_tma(x[k:k + 1].contiguous(), w, b, ln_stats=st1)
        assert torch.equal((st - pre)[k * H * W:(k + 1) * H * W], st1), f"ln_stats C={C}: image {k} differs from its B = 1 launch"


# ---------------------------------------------------------------------------------------------------------------- fused MLP
def gelu64(z):
    return 0.5 * z * (1 + torch.erf(z / math.sqrt(2)))


def mlp_operands(C, seed):
    g = G(seed)
    lw, lb = (1 + 0.2 * torch.randn(C, generator=g)).to(dev), (0.1 * torch.randn(C, generator=g)).to(dev)
    w1 = (torch.randn(4 * C, C, generator=g) / C ** 0.5).to(dev)
    b1 = (0.1 * torch.randn(4 * C, generator=g)).to(dev)
    w2 = (torch.randn(C, 4 * C, generator=g) / (4 * C) ** 0.5).to(dev)
    b2 = (0.1 * torch.randn(C, generator=g)).to(dev)
    gamma = (0.5 * torch.randn(C, generator=g)).to(dev)
    return dict(w1f=(w1 * lw[None, :]).bfloat16().contiguous(), c1=(w1 @ lb + b1).contiguous(), w2=w2.bfloat16().contiguous(), b2=b2,
                gamma=gamma)


def run_mlp(t, x, p):
    return ops.convnext_mlp(t, p["w1f"], p["c1"], p["w2"], p["b2"], p["gamma"], x, 1e-6)


def mlp_ref(t, x, p, drop_chunk=None):
    """The kernel's chain in float64 with its rounding points: tn = bf16(LN(t)), h = bf16(GELU(tn W1f^T + c1)),
    out = x + gamma (h W2^T + b2); and the per-element bound.  K = 4C, the hidden width.

      * GEMM2 in fp32: K u (|h| |W2|^T) (wgmma accumulates the K exact products, one rounding per step at worst);
      * continuous errors of z = tn W1f^T + c1, propagated through |GELU'| <= 1.13 and |W2| worst case: the fp32 LayerNorm (mean
        summed over C values in fp32: (C/2 + 1) u mean|t| before the scaling by rstd; scale and variance: (C/2 + 3) u |tn|), and
        GEMM1 in fp32 (C u |tn| |W1f|^T); plus the GELU fit, GELU_FIT sum |W2|;
      * one-ulp disagreements of the two bf16 intermediates (the kernel's fp32 value and the float64 one on different sides of
        a rounding tie): ulp(tn) propagated through W1f and GELU', plus ulp(h), propagated through W2 as a root sum of squares.
        These happen only near ties and with random sign; a worst-case sum would be sqrt(K) too loose to detect a dropped chunk;
      * the epilogue (acc + b2) * gamma + x in fp32: 2^-22 (|x| + |gamma| (|y| + |b2|)).
    drop_chunk = j leaves hidden units 64 j .. 64 j + 63 out of the reference (the non-vacuity check)."""
    C = t.shape[1]
    td = t.double()
    mean = td.mean(1, keepdim=True)
    var = ((td - mean) ** 2).mean(1, keepdim=True)
    rstd = (var + 1e-6).rsqrt()
    tn = ((td - mean) * rstd).bfloat16().double()
    W1, W2 = p["w1f"].double(), p["w2"].double()
    z = tn @ W1.t() + p["c1"].double()
    h = gelu64(z).bfloat16().double()
    if drop_chunk is not None:
        h[:, 64 * drop_chunk:64 * drop_chunk + 64] = 0
    y = h @ W2.t() + p["b2"].double()
    gm = p["gamma"].double()
    ref = x.double() + gm * y
    f = lambda v: v.float()  # noqa: E731  (bound terms need no float64 precision)
    aW1, aW2 = f(W1).abs(), f(W2).abs()
    K = 4 * C
    e_gemm2 = K * U * (f(h).abs() @ aW2.t())
    dmean = (C / 2 + 1) * U * f(td.abs().mean(1, keepdim=True) * rstd)
    e_z = dmean * aW1.sum(1) + (C + C / 2 + 3) * U * (f(tn).abs() @ aW1.t())
    e_cont = (GELU_DMAX * e_z + GELU_FIT) @ aW2.t()
    e_zflip = (f(ulp_bf16(tn)) ** 2 @ (f(W1) ** 2).t()).sqrt()
    e_flip = ((f(ulp_bf16(h)) + GELU_DMAX * e_zflip) ** 2 @ (f(W2) ** 2).t()).sqrt()
    e_epi = 2.0 ** -22 * (x.double().abs() + gm.abs() * (y.abs() + p["b2"].double().abs()))
    bound = ref.abs() * REL + gm.abs() * (e_gemm2 + e_cont + e_flip).double() + e_epi + 1e-6
    return ref, bound


MLP_C = [96, 192, 256, 384]


def multipass_rows():
    """2 row tiles per SM and a partial third: the persistent CTAs each run two or three tiles, reusing the row-tile buffer and the
    weight ring (C = 256: one row-tile buffer, refilled after the last GEMM1 of the previous tile)."""
    return 2 * torch.cuda.get_device_properties(0).multi_processor_count * 128 + 77


@pytest.mark.parametrize("C", MLP_C)
def test_convnext_mlp_rows_per_element(C):
    """Row counts around the 128-row tile and a multi-pass schedule, per element against float64; rows M onward of the buffer
    x lives in, and t, stay unchanged; the one-chunk-short reference fails the same check."""
    p = mlp_operands(C, 40 + C)
    for M in (1, 63, 64, 65, 127, 128, 129, multipass_rows()):
        g = G(M + C)
        t = (torch.randn(M, C, generator=g) * 1.5 + 0.3).to(dev).bfloat16()
        buf = torch.randn(M + 133, C, generator=g).to(dev).bfloat16()
        buf0, t0 = buf.clone(), t.clone()
        x0 = buf0[:M]
        out = run_mlp(t, buf[:M], p)
        ref, bound = mlp_ref(t, x0, p)
        check(out, ref, bound, f"convnext_mlp C={C} M={M}")
        assert torch.equal(buf[M:], buf0[M:]), f"convnext_mlp C={C} M={M}: guard rows past M overwritten"
        assert torch.equal(t, t0), f"convnext_mlp C={C} M={M}: t changed"
        if M == 129:
            ref_d, bound_d = mlp_ref(t, x0, p, drop_chunk=4 * C // 64 - 1)
            with pytest.raises(AssertionError):
                check(out, ref_d, bound_d, f"convnext_mlp C={C} M={M} vs reference without the last hidden chunk (must fail)")


@pytest.mark.parametrize("C", MLP_C)
def test_convnext_mlp_row_tiles_independent(C):
    """Rows of the first, a middle (the second of CTA 0) and the last, partial tile of the multi-pass run are bit for bit the
    rows of a run of that tile alone: no row-tile buffer or weight-ring stage leaks between the tiles of a persistent CTA."""
    p = mlp_operands(C, 50 + C)
    M = multipass_rows()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    g = G(C)
    t = (torch.randn(M, C, generator=g) * 1.5 + 0.3).to(dev).bfloat16()
    x = torch.randn(M, C, generator=g).to(dev).bfloat16()
    out = run_mlp(t, x.clone(), p)
    for tile in (0, sms, 2 * sms):
        r0, r1 = tile * 128, min(tile * 128 + 128, M)
        one = run_mlp(t[r0:r1].contiguous(), x[r0:r1].clone(), p)
        assert torch.equal(out[r0:r1], one), f"convnext_mlp C={C}: rows of tile {tile} differ from a run of that tile alone"


@pytest.mark.parametrize("ratio", [0, 100, 1000])
@pytest.mark.parametrize("C", MLP_C)
def test_convnext_mlp_special_rows(C, ratio):
    """ratio 0: constant rows of t (variance 0: tn = 0, the output is x + gamma (W2 bf16(GELU(c1)) + b2)), a different constant per
    row, zero included.  ratio 100 / 1000: rows with |mean| / std = ratio (bases 768 and -384, exact bf16 values); the in-kernel
    LayerNorm is two-pass over the bf16 values."""
    p = mlp_operands(C, 60 + C)
    M = 131
    g = G(ratio + C)
    if ratio == 0:
        t = (torch.arange(M, dtype=torch.float64)[:, None] / 8 - 8).expand(M, C)
    else:
        t = torch.stack([offset_values(C, 768.0 if r % 2 else -384.0, ratio, g) for r in range(M)])
        td = t.double()
        print(f"realised |mean|/std: {(td.mean(1).abs() / td.std(1, unbiased=False)).min().item():.0f} .. "
              f"{(td.mean(1).abs() / td.std(1, unbiased=False)).max().item():.0f}")
    t = t.to(dev).bfloat16().contiguous()
    x = torch.randn(M, C, generator=g).to(dev).bfloat16()
    out = run_mlp(t, x.clone(), p)
    ref, bound = mlp_ref(t, x, p)
    check(out, ref, bound, f"convnext_mlp C={C} special rows ratio={ratio}")


# ---------------------------------------------------------------------------------------------------------------- dwconv7 + LN
def dwln_target(B, H, W, C):
    """The kernel uc_dwconv7_ln dispatches to (launch_dwln): C % 64 != 0 -> dwconv7_ln_kernel; else the first dwln_kernel tile of
    16x8, 8x8, 8x4 whose [pixels][C] buffer fits 227 KB of shared memory and that gives at least 100 CTAs, else 4x2."""
    if C % 64:
        return "row"
    for TW, TH in ((16, 8), (8, 8), (8, 4)):
        smem = 2 * (TH + 6) * (TW + 6) * 128 + 2 * 49 * 64 * 4 + TW * TH * C * 2
        if smem <= 227 * 1024 and -(-W // TW) * -(-H // TH) * B >= 100:
            return f"{TW}x{TH}"
    return "4x2"


DWLN_SHAPES = [  # C, H, W, B
    (128, 41, 81, 3), (384, 100, 160, 1),                      # 16x8, partial tiles
    (128, 80, 80, 1), (512, 41, 81, 2),                        # 8x8 (too few 16x8 CTAs / 16x8 buffer too large)
    (64, 60, 60, 1), (1536, 40, 80, 1), (768, 50, 80, 1),      # 8x4
    (128, 7, 7, 3), (64, 1, 1, 1), (1536, 5, 9, 2), (192, 3, 2, 1),  # 4x2 (tiny maps)
    (96, 20, 28, 2), (200, 9, 17, 3), (1534, 5, 9, 1), (8, 1, 9, 1), (2, 3, 4, 2),  # dwconv7_ln_kernel
]
DWLN_TARGETS = {"16x8", "8x8", "8x4", "4x2", "row"}


def test_dwln_shapes_hit_every_target():
    hit = {dwln_target(B, H, W, C) for C, H, W, B in DWLN_SHAPES}
    assert hit == DWLN_TARGETS, hit


def dwln_ref(x, w, b, lnw, lnb):
    """float64 y = conv(x) + b, rounded to bf16 for the dwln_kernel tiles (the kernel parks the conv output as bf16 before the
    LayerNorm) and not for dwconv7_ln_kernel (which normalises the fp32 sum); out = LN(y) lnw + lnb, and the bound:

      * e_y, the error of the y the kernel normalises: 49 u S for the fp32 sum (see DW_C); for the rounding tiles one ulp(y), charged
        only where float64 y lies within 49 u S of a rounding tie (elsewhere the kernel's fp32 sum rounds to the same bf16 value);
      * its effect on the statistics: the mean moves by mean_c e_y, rstd by rstd mean_c(|tn| e_y) relatively;
      * the fp32 statistics: sums over C of chain length n = C/32 + 30 (lane loop, 5 shuffles, up to 24 warps): the mean is off
        by (n + 1) u mean|y|, the variance and rstd add (n + 6) u |tn|;
      * the affine epilogue in fp32: 2^-22 |lnb|."""
    B, H, W, C = x.shape
    y, S = dw_ref(x, w, b)
    if dwln_target(B, H, W, C) != "row":
        yq = y.bfloat16().double()
        acc = DW_C["tma"] * U * S
        # the nearest tie is half a gap away from yq, and the gap below a power of two is half the gap above it
        tie = (torch.minimum(ulp_bf16(yq), ulp_bf16(y)) / 2 - (y - yq).abs()) <= acc
        e_y = tie.double() * ulp_bf16(yq)
        y = yq
    else:
        e_y = DW_C["tma"] * U * S
    mean = y.mean(3, keepdim=True)
    rstd = (((y - mean) ** 2).mean(3, keepdim=True) + 1e-6).rsqrt()
    tn = (y - mean) * rstd
    lw, lb = lnw.double(), lnb.double()
    ref = tn * lw + lb
    n = C / 32 + 30
    e_tn = rstd * (e_y + e_y.mean(3, keepdim=True) + (n + 1) * U * y.abs().mean(3, keepdim=True)) \
        + tn.abs() * (rstd * (tn.abs() * e_y).mean(3, keepdim=True) + (n + 6) * U)
    bound = ref.abs() * REL + lw.abs() * e_tn + 2.0 ** -22 * lb.abs() + 1e-6
    return ref, bound


def dwln_params(C, g, scale=1.0):
    w = (torch.randn(C, 1, 7, 7, generator=g) / 7 * scale).to(dev)
    lnw, lnb = (1 + 0.3 * torch.randn(C, generator=g)).to(dev), (0.5 * torch.randn(C, generator=g)).to(dev)
    return w, lnw, lnb


def run_dwln(x, w, b, lnw, lnb, out=None):
    return ops.dwconv7_ln(x, ops.pack_dw_weight(w), b, lnw, lnb, 1e-6, out=out)


@pytest.mark.parametrize("C,H,W,B", DWLN_SHAPES)
def test_dwconv7_ln_targets(C, H, W, B):
    """Random maps per element against float64 on every dispatch target; the output is the first B images of a buffer with a guard
    image after them; a B > 1 launch gives each image the bits of its B = 1 launch when that selects the same target."""
    g = G(400 + C + H)
    x = torch.randn(B, H, W, C, generator=g).to(dev).bfloat16()
    w, lnw, lnb = dwln_params(C, g)
    b = torch.randn(C, generator=g).to(dev)
    buf = torch.randn(B + 1, H, W, C, generator=g).to(dev).bfloat16()
    buf0 = buf.clone()
    out = run_dwln(x, w, b, lnw, lnb, out=buf[:B])
    tgt = dwln_target(B, H, W, C)
    ref, bound = dwln_ref(x, w, b, lnw, lnb)
    check(out, ref, bound, f"dwconv7_ln [{tgt}] C={C} H={H} W={W} B={B}")
    assert torch.equal(buf[B], buf0[B]), f"dwconv7_ln C={C}: guard image overwritten"
    if B > 1 and dwln_target(1, H, W, C) == tgt:
        for k in range(B):
            assert torch.equal(out[k], run_dwln(x[k:k + 1].contiguous(), w, b, lnw, lnb)[0]), f"dwconv7_ln C={C}: image {k}"


def test_dwconv7_ln_rounding_point_is_pinned():
    """The two families round at different points, and the bound tells them apart: the 16x8 tile output fails the check against
    the unrounded (dwconv7_ln_kernel) reference where |mean| / std is large enough for one ulp of y to matter."""
    C, H, W, B = 128, 41, 81, 3
    g = G(11)
    x = (torch.randn(B, H, W, C, generator=g) * 0.1).to(dev).bfloat16()
    w, lnw, lnb = dwln_params(C, g)
    b = offset_values(C, 96.0, 100, g).float().to(dev)
    out = run_dwln(x, w, b, lnw, lnb)
    y, S = dw_ref(x, w, b)
    mean = y.mean(3, keepdim=True)
    rstd = (((y - mean) ** 2).mean(3, keepdim=True) + 1e-6).rsqrt()
    ref = (y - mean) * rstd * lnw.double() + lnb.double()
    with pytest.raises(AssertionError):
        check(out, ref, ref.abs() * REL + lnw.double().abs() * rstd * DW_C["tma"] * U * S + 1e-6,
              "dwconv7_ln 16x8 vs unrounded reference (must fail)")


@pytest.mark.parametrize("C,H,W,B", DWLN_SHAPES)
def test_dwconv7_ln_equal_channels(C, H, W, B):
    """Identical filters and biases over a map whose channels are equal at every pixel: all C conv outputs of a pixel are equal (and
    exact in fp32: products of k/8 and k/256), so the variance is 0 and the output must be lnb exactly (lnb exact in bf16 and
    >= 1 in magnitude, far from a rounding tie; rstd = 1/sqrt(eps) times a mean off by at most one fp32 ulp stays below it)."""
    g = G(500 + C)
    v = (torch.randint(-16, 17, (B, H, W, 1), generator=g).double() / 8).expand(B, H, W, C)
    x = v.contiguous().to(dev).bfloat16()
    w = (torch.randint(-8, 9, (1, 1, 7, 7), generator=g).double() / 256).expand(C, 1, 7, 7).contiguous().float().to(dev)
    b = torch.full((C,), 0.25, device=dev)
    lnw = (1 + 0.3 * torch.randn(C, generator=g)).to(dev)
    lnb = ((1 + torch.randint(0, 4, (C,), generator=g).double() / 4) * torch.where(torch.rand(C, generator=g) < 0.5, -1.0, 1.0))
    lnb = lnb.float().to(dev)
    out = run_dwln(x, w, b, lnw, lnb)
    want = lnb.bfloat16().expand(B, H, W, C)
    assert torch.equal(out, want), f"dwconv7_ln [{dwln_target(B, H, W, C)}] C={C}: equal channels give " \
                                   f"{(out != want).sum().item()} outputs != lnb"


@pytest.mark.parametrize("ratio", [100, 1000])
@pytest.mark.parametrize("C,H,W,B", [(128, 41, 81, 3), (128, 80, 80, 1), (64, 60, 60, 1), (128, 7, 7, 3), (96, 20, 28, 2)])
def test_dwconv7_ln_large_offset(C, H, W, B, ratio):
    """Conv outputs with |mean| / std ~ ratio over the channels of every pixel: biases offset_values(768, ratio) and a small
    convolution on top; the LayerNorm is two-pass in fp32 in both kernel families."""
    g = G(600 + C + ratio)
    x = torch.randn(B, H, W, C, generator=g).to(dev).bfloat16()
    w, lnw, lnb = dwln_params(C, g, scale=0.05)
    b = offset_values(C, 768.0, ratio, g).float().to(dev)
    out = run_dwln(x, w, b, lnw, lnb)
    y, _ = dw_ref(x, w, b)
    r = y.mean(3).abs() / y.std(3, unbiased=False)
    print(f"realised |mean|/std: {r.min().item():.0f} .. {r.max().item():.0f}")
    ref, bound = dwln_ref(x, w, b, lnw, lnb)
    check(out, ref, bound, f"dwconv7_ln [{dwln_target(B, H, W, C)}] C={C} |mean|/std={ratio}")


# ---------------------------------------------------------------------------------------------------------------- LayerNorm fold
LNFOLD_FLOOR = 1e-3  # as the GroupNorm chain (test_kernel_edges_gpu.GN_FLOOR): a quarter of a bf16 ulp at 0.5


def lnfold_chain(ratio, C, seed=17):
    """uc_dwconv7 with ln_stats, then uc_conv2d with row_stats (pwconv1 with the LayerNorm folded in, GELU).  The reference applies
    the exact float64 LayerNorm of the stored bf16 depthwise output, so the comparison measures the statistics path.  The bound:
    REL |ref| + LNFOLD_FLOOR + the GELU fit + |GELU'| <= 1.13 times the fp32 errors of the folded pre-activation
    rstd (W1f t) - rstd mu colsum(W1f) + c1: the GEMM over the un-normalised t (C u rstd |t| |W1f|^T) and the two products of
    the mean term (2^-22 rstd |mu| |colsum|).  colsum is the float64 column sum rounded once to fp32."""
    B, H, W = 2, 12, 20
    g = G(seed)
    x = torch.randn(B, H, W, C, generator=g).to(dev).bfloat16()
    wd = (torch.randn(C, 1, 7, 7, generator=g) / 7).to(dev)
    bd = (ratio + 0.1 * torch.randn(C, generator=g)).to(dev)
    lw, lb = (1 + 0.2 * torch.randn(C, generator=g)).to(dev), (0.1 * torch.randn(C, generator=g)).to(dev)
    w1 = (torch.randn(4 * C, C, generator=g) / C ** 0.5).to(dev)
    b1 = (0.1 * torch.randn(4 * C, generator=g)).to(dev)
    w1f = ops.pack_conv_weight((w1 * lw[None, :])[:, :, None, None])
    s1 = w1f.double().sum(dim=(1, 2)).float().contiguous()
    c1 = (w1 @ lb + b1).contiguous()
    st = torch.zeros(B * H * W, 2, dtype=torch.int64, device=dev)
    t = ops.dwconv7(x, ops.pack_dw_weight(wd), bd, ln_stats=st)
    got = ops.conv2d(t, w1f, 1, 1, bias=c1, act=ops.ACT_GELU, row_stats=st, col_s=s1, row_eps=1e-6)
    td = t.double().reshape(-1, C)
    mu = td.mean(1, keepdim=True)
    var = ((td - mu) ** 2).mean(1, keepdim=True)
    rstd = (var + 1e-6).rsqrt()
    W1 = w1f.double()[:, 0, :]
    ref = gelu64(((td - mu) * rstd) @ W1.t() + c1.double())
    e_z = C * U * rstd * (td.abs() @ W1.abs().t()) + 2.0 ** -22 * rstd * mu.abs() * s1.double().abs()
    bound = ref.abs() * REL + LNFOLD_FLOOR + GELU_FIT + GELU_DMAX * e_z
    r = (mu.abs() / var.sqrt()).squeeze(1)
    err = (got.double().reshape(-1, 4 * C) - ref).abs()
    worst = (err / bound).max().item()
    print(f"err/bound {worst:.3f}  dwconv7 ln_stats -> conv2d row_stats chain C={C} |mean|/std={ratio} "
          f"(realised {r.min().item():.0f} .. {r.max().item():.0f})")
    return worst


@pytest.mark.parametrize("ratio", [0, 10, 100])
@pytest.mark.parametrize("C", [96, 192])
def test_lnfold_chain(C, ratio):
    """|mean| / std up to 100 holds to float64 within one bf16 rounding."""
    assert lnfold_chain(ratio, C) <= 1.0


@pytest.mark.xfail(strict=True, reason="the statistics are one-pass fixed-point sums of fp32 partial sums and squares, and the fold takes "
                                      "var = E[y^2] - mu^2 in fp32: at |mean| / std = 1000 the variance keeps only a few correct bits "
                                      "(err / bound 5.3 at C = 96 and 57 at C = 192 on an H100 80GB HBM3 at 700 W)")
@pytest.mark.parametrize("C", [96, 192])
def test_lnfold_chain_offset_1000(C):
    assert lnfold_chain(1000, C) <= 1.0

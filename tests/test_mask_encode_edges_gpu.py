"""The VOS result assembly (uc_vos_aggregate / _batched), the MOTS and BDD mask encoder (uc_mots_encode / _batched) and the COCO
instance encoder (uc_inst_encode_batched) bit for bit against their host definitions, at their word, chunk, run and cover edges.

Exact lattice.  Mask values are multiples of 2^-8 in [0, 1].  The frame resize F.interpolate(scale_factor=1/r, bilinear,
align_corners=False) at r in {0.5, 1, 1.5, 2} has the source scale float(1 / (1/r)) = r, so the source coordinate (i + 0.5) r - 0.5
and every bilinear fraction are multiples of 1/4; aligned_bilinear at f in {1, 2, 4, 8} has fractions k / f, multiples of 1/8.
Every product and partial sum of the upsample and the resize is then a multiple of 2^-8 2^-6 2^-4 = 2^-18 of magnitude <= 1 (the
weights are convex), i.e. an integer below 2^18 times 2^-18, which float32 holds exactly.  So the kernels' fp32 arithmetic is exact
in any order and any contraction, and must equal the float64 reference: the CPU test test_lattice_is_exact_in_float32 checks
this for every (r, f) used, with F.interpolate in float32 and float64 and with a float32 emulation of the kernels' operation
order, and that is what licenses == on the GPU.  Two thresholds: 0.5 on the grid, with pixels exactly at it (the strict >), and
0.3 off it (the production mask_thres).  The VOS background product prod(1 - m) is not exact on the lattice; it is the float32
product in list order (unicorn_vos.py:105-121), which the reference computes the same way, one rounding per step.

Outputs are discrete (labels, RLE strings) and are compared for equality: strings, offsets, emit flags, label maps and soft
masks.  The references are results.overlap_free and results.rle_encode (the MOTS evaluator's overlap removal and pycocotools'
compressed RLE), the VOS aggregation restated literally from the reference model (a mask_merge channel per object id, channel 0
the background, numpy argmax: the lowest channel wins ties), and for the instance encoder aligned_bilinear restated in float64 by
test_sampling_edges_gpu.ab_upsample.

The RLE encoder's integer logic is driven to its edges with masks built from explicit column-major boundary positions: frames
under 32 rows and one column wide, word counts just under, at and over 1024 (the scan's thread count) and 1080 x 1920; chunks of
ceil(words / 1024) words holding 0, 1, 2, 3 and >= 4 boundaries in every predecessor / successor combination (every branch of
run_cat in the scan); counts whose deltas c_i - c_{i-2} sit on both sides of every char-width edge; the first and the last pixel
set.  The capacity clip is checked at 0, inside a multi-char count, at a string boundary, at total - 1 and at total.

Off the lattice, the instance encoder's own sampling (final_up_at, resize_mix in mask.cu) must reproduce what
mask_final_up_kernel stores and what mots_planes_kernel samples, bit for bit.  At r = 1 the resize is the identity, so the fused
bit is exactly stored > thr; thresholds are taken from stored's own values (and one float below them), so pixels sit exactly at
thr and any last-ulp difference of the upsample flips a bit.  At r != 1 the fused strings must equal uc_mots_encode of the stored
masks, at thresholds taken from a float32 emulation of the documented operation order (fma as an exact float64 product plus the
addend, rounded once to float32).

Every check prints its number of exact comparisons, and every coverage claim (pixels at the threshold, ties, seam combinations,
char widths, short covers) is asserted on the data."""
import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from unicorn_b200 import _lib, ops, post_ops
from unicorn_b200 import results as R
from test_sampling_edges_gpu import G, MASK_MAPS, ab_upsample, edge_anchors, mask_case

gpu = pytest.mark.gpu
dev = "cuda"
f64 = torch.float64
RATIOS = (0.5, 1.0, 1.5, 2.0)
FACTORS = (1, 2, 4, 8)
THRS = (0.5, 0.3)
SENT = 0xA5  # chars past the capacity keep this byte
SCAN = 1024  # threads of the run scan (kMotsThreads)


def thr32(thr):
    return float(np.float32(thr))


def exact(n, name):
    print(f"{n} exact comparisons  {name}")
    assert n > 0, f"{name}: nothing compared"
    return n


def rng(seed):
    return np.random.default_rng(seed)


# ================================================================================================ references
def resize64(v, r, H, W):
    """F.interpolate(scale_factor=1/r, bilinear, align_corners=False)[..., :H, :W] in float64 on the CPU; v [..., Hin, Win]."""
    x = v.detach().cpu().double()
    lead = x.shape[:-2]
    out = F.interpolate(x.reshape(-1, 1, *x.shape[-2:]), scale_factor=1 / r, mode="bilinear", align_corners=False)[..., :H, :W]
    return out.reshape(*lead, *out.shape[-2:])


def cover(Hin, Win, H, W, r):
    """The hm x wm corner of an H x W frame that the resize covers (floor(in * (1/r)) in double precision)."""
    sf = 1.0 / r
    return min(H, int(math.floor(Hin * sf))), min(W, int(math.floor(Win * sf)))


def mots_ref(masks, order, emit, thr, r, H, W):
    """The MOTS evaluator's strings: rows outside [0, n_max) are empty masks; resize, threshold, overlap free in list order, then
    the strings of the emitted instances ("" for the others).  Returns (strings, resized values, overlap-free bits)."""
    n_max, Hin, Win = masks.shape
    if not order:
        return [], None, None
    zero = torch.zeros(Hin, Win, dtype=masks.dtype, device=masks.device)
    v = resize64(torch.stack([masks[o] if 0 <= o < n_max else zero for o in order]), r, H, W)
    free = R.overlap_free(v > thr32(thr)).numpy()
    return [R.rle_encode(free[i]) if emit[i] else "" for i in range(len(order))], v, free


def rle_counts(bits):
    """The COCO counts of a bool [H, W] mask (column-major runs, the first run counting zeros), as rle_encode forms them."""
    flat = np.asarray(bits, dtype=bool).reshape(-1, order="F")
    bounds = np.concatenate([[0], np.flatnonzero(flat[1:] != flat[:-1]) + 1, [flat.size]])
    c = np.diff(bounds)
    return np.concatenate([[0], c]) if flat[0] else c


def char_widths(s):
    """(chars per count, sign of each delta) of an RLE string: a count ends at a char without the continuation bit 0x20, and its
    delta is negative when that char's bit 0x10 is set."""
    widths, signs, w = [], [], 0
    for ch in s:
        c = ord(ch) - 48
        w += 1
        if not c & 0x20:
            widths.append(w)
            signs.append(-1 if c & 0x10 else 1)
            w = 0
    assert w == 0, "unterminated count"
    return widths, signs


def vos_ref(objs, Hin, Win, H, W, r):
    """unicorn_vos.py:129-155 + :105-121: every object's soft mask in the H x W frame (the resized network mask in the corner it
    covers, zeros beyond; or label == id for an initial label map), the float32 background product in list order, and numpy's
    argmax over mask_merge (channel 0 the background, channel id the object): the lowest channel wins ties."""
    n = len(objs)
    soft = torch.zeros(n, H, W, dtype=f64)
    for k, (oid, m, lab) in enumerate(objs):
        if lab is not None:
            soft[k] = (lab.cpu() == oid).double()
        elif m is not None:
            v = resize64(m, r, H, W)
            soft[k, :v.shape[0], :v.shape[1]] = v
    s32 = soft.float()
    assert torch.equal(s32.double(), soft), "the soft masks are not on the lattice"
    bg = torch.ones(H, W, dtype=torch.float32)
    for k in range(n):
        bg = bg * (1 - s32[k])
    merge = np.zeros((H, W, max(o[0] for o in objs) + 1))
    for k, (oid, _, _) in enumerate(objs):
        merge[:, :, oid] = s32[k].numpy()
    merge[:, :, 0] = bg.numpy()
    return s32, np.argmax(merge, axis=-1).astype(np.uint8), merge


def tie_counts(merge, ids):
    """Pixels where the background ties the best object, where >= 2 and >= 3 objects tie for the maximum above the background,
    and where >= 2 objects tie at 1.0."""
    obj = merge[:, :, sorted(set(ids))]
    best = obj.max(-1)
    nbest = (obj == best[..., None]).sum(-1)
    bg = merge[:, :, 0]
    return dict(bg_tie=int(((bg == best) & (best > 0)).sum()), two=int(((nbest >= 2) & (best > bg)).sum()),
                three=int(((nbest >= 3) & (best > bg)).sum()), saturated=int(((nbest >= 2) & (best == 1.0)).sum()))


# ================================================================================================ float32 emulation of mask.cu
def fma32(a, b, c):
    """fmaf: the product of two floats is exact in float64; the addend is added and the sum rounded once to float32."""
    return (a.double() * b.double() + c.double()).float()


def ab_taps32(n_out, f, n):
    """ab_coord: i0 = max(i - f/2, 0) div f, the fraction (k / f in float32: for a power of two, k * (1/f) is the same float)."""
    i = torch.arange(n_out)
    ii = (i - f // 2).clamp(min=0)
    i0 = ii // f
    frac = (ii - i0 * f).float() / f
    return i0.clamp(max=n - 1), (i0 + 1).clamp(max=n - 1), frac


def final_up_emul(s, f):
    """final_up_at (and, by its SASS, mask_final_up_kernel) on s float32 [n, hs, ws]: per source row fma(fx, right, (1 - fx) left),
    then fma(1 - fy, top, fy bot)."""
    _, hs, ws = s.shape
    y0, y1, fy = ab_taps32(hs * f, f, hs)
    x0, x1, fx = ab_taps32(ws * f, f, ws)
    gx = 1 - fx

    def row(y):
        t = s[:, y]
        return fma32(fx, t[:, :, x1], gx * t[:, :, x0])
    fy = fy[:, None]
    return fma32(1 - fy, row(y0), fy * row(y1))


def resize_taps32(n_out, n_in, scale):
    """resize_src: (i + 0.5) scale - 0.5 rounded once (the contracted fma), clamped at 0; i0, i1 and l = f - i0 in float32."""
    i = torch.arange(n_out, dtype=f64)
    src = ((i + 0.5) * float(scale) - 0.5).float().clamp(min=0)
    i0 = src.long().clamp(max=n_in - 1)
    return i0, (i0 + 1).clamp(max=n_in - 1), src - i0.float()


def resize_emul(t, r, H, W):
    """resize_mix of the four taps of the frame resize on t float32 [n, Hin, Win] -> [n, hm, wm]."""
    _, Hin, Win = t.shape
    hm, wm = cover(Hin, Win, H, W, r)
    scale = np.float32(1.0 / (1.0 / r))
    y0, y1, ly = resize_taps32(hm, Hin, scale)
    x0, x1, lx = resize_taps32(wm, Win, scale)
    top_r, bot_r = t[:, y0], t[:, y1]
    gx = 1 - lx
    top = fma32(gx, top_r[:, :, x0], lx * top_r[:, :, x1])
    bot = fma32(gx, bot_r[:, :, x0], lx * bot_r[:, :, x1])
    ly = ly[:, None]
    return fma32(1 - ly, top, ly * bot)


# ================================================================================================ inputs
def lattice(bits, thr, g):
    """Values on the 2^-8 grid for bool bits: set pixels above thr, clear pixels at or below it; a quarter of each sits on the grid
    point next to thr (exactly thr for thr = 0.5), a quarter at 1.0 / 0.0."""
    t = int(math.floor(thr32(thr) * 256))  # the largest grid index <= thr
    u = torch.randint(0, 4, bits.shape, generator=g)
    on = torch.randint(t + 1, 257, bits.shape, generator=g)
    on = torch.where(u == 0, t + 1, torch.where(u == 1, 256, on))
    off = torch.randint(0, t + 1, bits.shape, generator=g)
    off = torch.where(u == 0, t, torch.where(u == 1, 0, off))
    return torch.where(bits, on, off).float() / 256


def grid_values(shape, g, lo=0, hi=256):
    return torch.randint(lo, hi + 1, shape, generator=g).float() / 256


def bits_of(pos, H, W):
    """The bool [H, W] mask whose column-major bit changes (pixel -1 counting as 0) are exactly at the pixels `pos`."""
    flat = np.zeros(H * W, dtype=np.int64)
    flat[np.asarray(pos, dtype=np.int64)] = 1
    return torch.from_numpy((np.cumsum(flat) & 1).astype(bool).reshape(W, H).T.copy())


def words_of(H, W):
    """First pixel and rows of every 32-row word (words never straddle a column), and the scan's chunk of words per thread."""
    hw32 = -(-H // 32)
    w = np.arange(W * hw32)
    x, wy = w // hw32, w % hw32
    return x * H + 32 * wy, np.minimum(32, H - 32 * wy), -(-(W * hw32) // SCAN)


SEAM = [v for a in range(5) for b in range(5) for v in (a, b)]  # consecutive entries hold every (a, b) pair, 4 standing for >= 4


def seam_positions(H, W, rg):
    """Boundary pixels putting SEAM[t % 50] boundaries (4: 4 to 9) into chunk t of the scan, as many as its pixels allow."""
    start, rows, chunk = words_of(H, W)
    pos = []
    for t in range(-(-len(start) // chunk)):
        s, m = start[t * chunk:(t + 1) * chunk], rows[t * chunk:(t + 1) * chunk]
        want = SEAM[t % len(SEAM)]
        k = min(want if want < 4 else 4 + int(rg.integers(0, 6)), int(m.sum()))
        idx = np.sort(rg.choice(int(m.sum()), k, replace=False))
        end = np.cumsum(m)
        j = np.searchsorted(end, idx, side="right")
        pos.append(s[j] + idx - (end[j] - m[j]))
    return np.sort(np.concatenate(pos))


def seam_pairs(bits):
    """The (min(a, 4), min(b, 4)) boundary counts of consecutive scan chunks of a bool [H, W] mask."""
    H, W = bits.shape
    flat = np.asarray(bits, dtype=bool).reshape(-1, order="F")
    p = np.flatnonzero(flat != np.concatenate([[False], flat[:-1]]))
    hw32 = -(-H // 32)
    _, _, chunk = words_of(H, W)
    n = np.minimum(np.bincount((p // H * hw32 + p % H // 32) // chunk, minlength=SCAN), 4)
    return set(zip(n[:-1].tolist(), n[1:].tolist()))


DELTAS = (15, 16, 17, 511, 512, 513, 16383, 16384, 16385, 524287, 524288, 524289)


def delta_counts(P):
    """Counts with the first run empty (the first pixel set) and, for every d of DELTAS that fits, the runs 1, 1, 1 + d, 1, 1: the
    count 1 + d has delta +d and the count two after it -d.  The last run fills the frame."""
    c, left = [0, 7, 3], P - 10 - 1
    for d in DELTAS:
        if d + 5 <= left:
            c += [1, 1, 1 + d, 1, 1]
            left -= d + 5
    c.append(P - sum(c))
    assert c[-1] >= 1
    return c


# ================================================================================================ launches
def strings_of(chars, offsets, k, cap):
    """The k strings of one encode; the offsets must be complete and every char past the capacity untouched."""
    offs = offsets.cpu().tolist()[:k + 1]
    assert offs[0] == 0 and all(a <= b for a, b in zip(offs, offs[1:])), offs
    assert offs[-1] <= cap, f"{offs[-1]} chars do not fit the capacity {cap}"
    assert bool((chars[cap:] == SENT).all()), "chars past the capacity were written"
    s = bytes(chars[:offs[-1]].cpu().numpy()).decode("ascii")
    return [s[offs[i]:offs[i + 1]] for i in range(k)], offs


def mots_run(masks, order, emit, thr, r, H, W, cap):
    k = len(order)
    ws = ops.mots_encode_workspace(k, H, W, dev)
    chars = torch.full((cap + 256,), SENT, dtype=torch.uint8, device=dev)
    offsets = torch.full((k + 1,), -1, dtype=torch.int64, device=dev)
    ops.mots_encode(masks, torch.tensor(order, dtype=torch.int32, device=dev), torch.tensor([int(e) for e in emit], dtype=torch.uint8, device=dev),
                    thr, r, H, W, ws, chars[:cap], offsets)
    torch.cuda.synchronize()
    return strings_of(chars, offsets, k, cap)


def mots_check(masks, order, emit, thr, r, H, W, name):
    want, v, free = mots_ref(masks, order, emit, thr, r, H, W)
    got, _ = mots_run(masks, order, emit, thr, r, H, W, sum(map(len, want)) + 64)
    assert got == want, f"{name}: first differing string {next(i for i in range(len(want)) if got[i] != want[i])}"
    return want, v, free


def inst_run(maps, count, row0, f, thr, r, H, W, cap):
    B, n_max = maps.shape[:2]
    K = B * n_max
    ws = ops.mots_encode_workspace(K, max(H), max(W), dev)
    emit = torch.full((K,), 7, dtype=torch.uint8, device=dev)
    chars = torch.full((cap + 256,), SENT, dtype=torch.uint8, device=dev)
    offsets = torch.full((K + 1,), -1, dtype=torch.int64, device=dev)
    post_ops.inst_encode(maps, torch.tensor(count, dtype=torch.int32, device=dev), row0, f, thr, r, H, W, ws, emit, chars[:cap], offsets)
    torch.cuda.synchronize()
    got, _ = strings_of(chars, offsets, K, cap)
    return got, emit.cpu().tolist()


def vos_objects(objs):
    arr = (_lib.UcVosObject * len(objs))()
    for k, (oid, m, lab) in enumerate(objs):
        arr[k].id = oid
        arr[k].mask = m.data_ptr() if m is not None else None
        arr[k].init_mask = lab.data_ptr() if lab is not None else None
    return arr


def vos_run(videos, Hin, Win, batched):
    """videos: dicts (objs [(id, network mask [Hin, Win] or None, label map [H, W] or None)], H, W, r, soft); soft planes start at a
    sentinel, so an unwritten plane shows."""
    outs, keep = [], []
    descs = (_lib.UcVosVideo * len(videos))()
    for b, v in enumerate(videos):
        n = len(v["objs"])
        soft = torch.full((n, v["H"], v["W"]), -3.0, device=dev) if v["soft"] else None
        seg = torch.full((v["H"], v["W"]), 77, dtype=torch.uint8, device=dev)
        arr = vos_objects(v["objs"])
        keep.append(arr)
        outs.append((soft, seg))
        descs[b].objs = ctypes.cast(arr, ctypes.POINTER(_lib.UcVosObject))
        descs[b].n, descs[b].H, descs[b].W, descs[b].r = n, v["H"], v["W"], float(v["r"])
        descs[b].soft_out, descs[b].seg_out = ops._p(soft), ops._p(seg)
    if batched:
        _lib.check(ops._L().uc_vos_aggregate_batched(descs, len(videos), Hin, Win, ops._S()), "uc_vos_aggregate_batched")
    else:
        for b, v in enumerate(videos):
            soft, seg = outs[b]
            _lib.check(ops._L().uc_vos_aggregate(keep[b], len(v["objs"]), Hin, Win, v["H"], v["W"], ctypes.c_float(v["r"]), ops._p(soft),
                                                 ops._p(seg), ops._S()), "uc_vos_aggregate")
    torch.cuda.synchronize()
    return outs


def vos_check(videos, Hin, Win, batched, name):
    outs = vos_run(videos, Hin, Win, batched)
    n_cmp, ties = 0, dict(bg_tie=0, two=0, three=0, saturated=0)
    for b, (v, (soft, seg)) in enumerate(zip(videos, outs)):
        s_ref, seg_ref, merge = vos_ref(v["objs"], Hin, Win, v["H"], v["W"], v["r"])
        got = seg.cpu().numpy()
        assert np.array_equal(got, seg_ref), f"{name} video {b}: {int((got != seg_ref).sum())} labels differ"
        n_cmp += got.size
        if soft is not None:
            assert torch.equal(soft.cpu(), s_ref), f"{name} video {b}: soft masks differ"
            n_cmp += s_ref.numel()
        for key, val in tie_counts(merge, [o[0] for o in v["objs"]]).items():
            ties[key] += val
    exact(n_cmp, f"{name} (labels + soft values; ties {ties})")
    return ties


# ================================================================================================ CPU: the lattice and the references
def test_lattice_is_exact_in_float32():
    """On the 2^-8 grid, at every (r, f) the GPU tests use: F.interpolate in float32 equals float64; aligned_bilinear (ab_upsample in
    float64) equals its float32 emulation in the kernels' operation order, and so does the resize of that; every value is a multiple
    of 2^-18 in [0, 1]."""
    g = G(11)
    n = 0
    for hs, ws in ((7, 5), (12, 10), (2, 3)):
        t = grid_values((3, hs, ws), g)
        for r in RATIOS:
            H, W = 4 * hs, 4 * ws
            a, b = resize64(t, r, H, W), F.interpolate(t[:, None], scale_factor=1 / r, mode="bilinear", align_corners=False)[:, 0, :H, :W]
            assert torch.equal(a, b.double()), (hs, ws, r)
            assert torch.equal(resize_emul(t, r, H, W).double(), a), (hs, ws, r)
            n += a.numel()
        for f in FACTORS:
            up = ab_upsample(t, f)
            up32 = final_up_emul(t, f)
            assert torch.equal(up32.double(), up), (hs, ws, f)
            assert torch.equal(up * 2 ** 14, torch.round(up * 2 ** 14)) and up.min() >= 0 and up.max() <= 1
            for r in RATIOS:
                H, W = hs * f * 2, ws * f * 2
                v = resize64(up, r, H, W)
                v32 = F.interpolate(up32[:, None], scale_factor=1 / r, mode="bilinear", align_corners=False)[:, 0, :H, :W]
                assert torch.equal(v32.double(), v), (hs, ws, f, r)
                assert torch.equal(resize_emul(up32, r, H, W).double(), v), (hs, ws, f, r)
                assert torch.equal(v * 2 ** 18, torch.round(v * 2 ** 18))
                n += 2 * v.numel()
    exact(n, "lattice: float32 == float64")


def test_short_covers_and_source_scales():
    """The covers the GPU tests rely on: r = 800/402 gives 401 rows from 800 (one short of the frame), the lattice ratios have an
    exact source scale float(1 / (1/r)) == r and never floor one short."""
    x = torch.zeros(1, 1, 800, 80)
    assert F.interpolate(x, scale_factor=1 / (800 / 402), mode="bilinear", align_corners=False).shape[2] == 401
    assert cover(800, 80, 402, 41, 800 / 402) == (401, 40)
    for r in RATIOS:
        assert float(np.float32(1.0 / (1.0 / r))) == r
        for n in range(1, 2000):
            assert cover(n, n, 10 ** 6, 10 ** 6, r)[0] == math.floor(n / r)


def test_references_pin_the_definitions():
    """The reference helpers against hand-worked cases: rle_counts and char_widths agree with rle_encode / rle_decode; the VOS
    argmax gives background ties to the background and object ties to the lower id whatever the list order; bits_of puts the
    changes where asked; out-of-range rows are empty masks."""
    g = G(12)
    for H, W in ((1, 1), (3, 5), (33, 2)):
        for _ in range(20):
            m = torch.rand(H, W, generator=g) < 0.5
            s = R.rle_encode(m.numpy())
            assert np.array_equal(R.rle_decode(s, H, W), m.numpy())
            c = rle_counts(m.numpy())
            widths, _ = char_widths(s)
            assert len(widths) == len(c) and c.sum() == H * W
    assert char_widths(R.rle_encode(np.ones((3, 2), bool))) == ([1, 1], [1, 1])  # counts 0, 6
    for d, w in ((15, 1), (16, 2), (-16, 1), (-17, 2), (511, 2), (512, 3), (-512, 2), (-513, 3), (16383, 3), (16384, 4), (-16384, 3),
                 (-16385, 4), (524287, 4), (524288, 5), (-524288, 4), (-524289, 5)):
        x, n, more = d, 0, True
        while more:  # rleToString's char loop
            ch = x & 0x1F
            x >>= 5
            more = (x != -1) if ch & 0x10 else (x != 0)
            n += 1
        assert n == w, (d, n, w)
    pos = [0, 5, 6, 14]
    b = bits_of(pos, 4, 4).numpy().reshape(-1, order="F")
    assert np.flatnonzero(b != np.concatenate([[False], b[:-1]])).tolist() == pos
    half = torch.full((4, 4), 0.5)
    _, seg, _ = vos_ref([(3, half, None)], 4, 4, 4, 4, 1.0)
    assert (seg == 0).all()  # background 0.5 ties the object
    tq = torch.full((4, 4), 0.75)
    _, seg, _ = vos_ref([(9, tq, None), (3, tq, None), (5, tq, None)], 4, 4, 4, 4, 1.0)
    assert (seg == 3).all()
    want, _, _ = mots_ref(torch.ones(2, 3, 3), [-1, 2, 0], [1, 1, 1], 0.5, 1.0, 3, 3)
    assert want == [R.rle_encode(np.zeros((3, 3), bool))] * 2 + [R.rle_encode(np.ones((3, 3), bool))]


def test_generators_reach_their_edges():
    """The boundary generators produce what the GPU tests claim, before any kernel runs: every chunk-seam combination on the seam
    frames, every char width and negative deltas."""
    for H, W in SEAM_FULL:
        pos = seam_positions(H, W, rng(H * 7 + W))
        assert seam_pairs(bits_of(pos, H, W).numpy()) == {(a, b) for a in range(5) for b in range(5)}, (H, W)
    c = delta_counts(1080 * 1920)
    deltas = [c[i] - c[i - 2] for i in range(3, len(c))]
    assert all(d in deltas and -d in deltas for d in DELTAS)


# ================================================================================================ uc_mots_encode
FRAMES = [(1, 1), (1, 2), (1, 1025), (31, 33), (32, 1023), (32, 1024), (32, 1025), (33, 512), (64, 1), (64, 512), (65, 341), (401, 79),
          (401, 2), (1080, 1920)]
SEAM_FULL = [(32, 1023), (32, 1024), (32, 1025), (64, 512), (401, 79), (1080, 1920)]  # every chunk can hold >= 4 boundaries


@gpu
@pytest.mark.parametrize("thr", THRS)
@pytest.mark.parametrize("hm,wm", FRAMES)
def test_mots_encode_boundary_lattice(hm, wm, thr):
    """r = 1 (the resize is the identity): masks from explicit boundary lists at frames 1 row high, 1 or 2 columns wide, under,
    at and over 1024 words and 1080 x 1920: two chunk-seam masks, the first pixel alone, the last pixel alone, full, empty and random
    bits (small frames), all in one overlapping encode and each alone.  Values are lattice() of the bits, so pixels sit exactly on
    thr = 0.5."""
    rg, g = rng(hm * 31 + wm), G(hm * 17 + wm)
    P = hm * wm
    bits = [bits_of(seam_positions(hm, wm, rg), hm, wm), bits_of([0] + ([1] if P > 1 else []), hm, wm), bits_of([P - 1], hm, wm),
            torch.ones(hm, wm, dtype=torch.bool), torch.zeros(hm, wm, dtype=torch.bool), bits_of(seam_positions(hm, wm, rg), hm, wm)]
    if P <= 70000:
        bits.append(torch.rand(hm, wm, generator=g) < 0.5)
    masks = torch.stack([lattice(b, thr, g) for b in bits])
    masks[4] = math.floor(thr32(thr) * 256) / 256  # the empty mask on the grid point at or below thr: exactly thr for 0.5
    masks = masks.to(dev)
    assert thr != 0.5 or bool((masks[4] == 0.5).all())
    n = len(bits)
    order = [0, 5, 1, 2] + list(range(6, n)) + [3, 4]
    want, _, free = mots_check(masks, order, [1] * n, thr, 1.0, hm, wm, f"{hm}x{wm} all")
    cmp = len(want)
    if (hm, wm) in SEAM_FULL:
        pairs = seam_pairs(free[0])
        assert pairs == {(a, b) for a in range(5) for b in range(5)}, sorted(pairs)
    for i in range(n):
        w, _, _ = mots_check(masks, [i], [1], thr, 1.0, hm, wm, f"{hm}x{wm} row {i}")
        assert w == [R.rle_encode(bits[i].numpy())]  # the lattice values threshold back to the bits
        cmp += 1
    exact(cmp, f"mots boundary lattice {hm}x{wm} thr={thr} (strings; seam pairs {len(seam_pairs(free[0]))}/25)")


@gpu
@pytest.mark.parametrize("hm,wm", [(1080, 1920), (401, 79)])
def test_mots_encode_count_deltas_at_char_widths(hm, wm):
    """Counts whose deltas c_i - c_{i-2} are +-15/16/17, +-511/512/513, +-16383/16384/16385 and +-524287/524288/524289 (as many as
    the frame holds), with the first pixel set: every char width the frame allows (1-5 at 1080 x 1920) and negative deltas occur."""
    g = G(hm + wm)
    c = delta_counts(hm * wm)
    bits = bits_of(np.cumsum(c)[:-1], hm, wm)
    masks = torch.stack([lattice(bits, 0.5, g), lattice(~bits, 0.5, g)]).to(dev)
    want, _, _ = mots_check(masks, [0], [1], 0.5, 1.0, hm, wm, f"deltas {hm}x{wm}")
    want2, _, _ = mots_check(masks, [1], [1], 0.5, 1.0, hm, wm, f"deltas {hm}x{wm} inverted")
    widths, signs = char_widths(want[0])
    assert np.array_equal(rle_counts(bits.numpy()), np.array(c))
    assert bool(bits[0, 0]) and not bool(masks[1, 0, 0] > 0.5)
    top = 5 if hm * wm > 2 * 524289 else 3
    assert set(range(1, top + 1)) <= set(widths) and -1 in signs, (sorted(set(widths)), set(signs))
    exact(2, f"mots count deltas {hm}x{wm} (widths {sorted(set(widths))}, {signs.count(-1)} negative deltas)")


@gpu
@pytest.mark.parametrize("r", (1.0, 1.5))
@pytest.mark.parametrize("thr", THRS)
@pytest.mark.parametrize("Hin,Win", [(65, 97), (401, 79)])
def test_mots_encode_overlap_removal(Hin, Win, thr, r):
    """Random bits at densities 0.5 and 0.05, heavily overlapping rectangles, a full and an empty mask; order rows -1, n_max and
    99 (empty masks) and a repeated row; emit = 0 instances still claim their pixels."""
    g = G(Hin + Win + int(10 * r))
    n_max = 12
    bits = [torch.rand(Hin, Win, generator=g) < d for d in (0.5, 0.5, 0.5, 0.05, 0.05, 0.05)]
    for s in range(3):
        b = torch.zeros(Hin, Win, dtype=torch.bool)
        b[Hin // 5 + s:Hin // 2 + 2 * s, Win // 6 + s:Win // 2 + s] = True
        bits.append(b)
    bits += [torch.ones(Hin, Win, dtype=torch.bool), torch.zeros(Hin, Win, dtype=torch.bool), torch.rand(Hin, Win, generator=g) < 0.5]
    masks = torch.stack([lattice(b, thr, g) for b in bits]).to(dev)
    order = [6, 2, -1, 7, 0, n_max, 8, 3, 9, 4, 99, 6]
    emit = [1, 1, 1, 0, 1, 1, 1, 0, 1, 1, 1, 1]
    H, W = cover(Hin, Win, 10 ** 6, 10 ** 6, r)
    want, v, free = mots_check(masks, order, emit, thr, r, H, W, f"overlap {Hin}x{Win} r={r}")
    raw = (v > thr32(thr)).numpy()
    assert (raw[1:] & ~free[1:]).any(), "no pixel was removed by the overlap"
    assert (raw[3] & raw[6]).any() and not (free[6] & raw[3]).any(), "a non-emitted instance must still claim its pixels"
    assert want[2] == want[5] == want[10] == R.rle_encode(np.zeros((H, W), bool))
    if thr == 0.5:
        assert int((v == 0.5).sum()) > 0
    exact(len(want), f"mots overlap {Hin}x{Win} thr={thr} r={r}")


def blocky(n, Hin, Win, g, k=3):
    """Lattice masks of k x k blocks of grid values, with the top eighth of the rows exactly 0.5 and below it a saturated and an
    empty block."""
    m = grid_values((n, -(-Hin // k), -(-Win // k)), g)
    m = m.repeat_interleave(k, 1).repeat_interleave(k, 2)[:, :Hin, :Win].contiguous()
    e = max(1, Hin // 8)
    m[:, :e] = 0.5
    m[:, e:2 * e + 1, :Win // 3] = 1.0
    m[:, e:2 * e + 1, Win // 3:2 * Win // 3] = 0.0
    return m


@gpu
@pytest.mark.parametrize("thr", THRS)
@pytest.mark.parametrize("r", (0.5, 1.5, 2.0))
def test_mots_encode_resize_lattice(r, thr):
    """r != 1 on the lattice: the resized values are exact, so every string must equal the host path's; frames covered exactly,
    cropped, and larger than the cover (hm x wm < H x W), at 45 x 37 and at 300 x 200 (over 1024 words at r = 0.5)."""
    cmp, at_thr = 0, 0
    for Hin, Win in ((45, 37), (300, 200)):
        g = G(int(r * 100) + Hin)
        masks = blocky(6, Hin, Win, g).to(dev)
        hc, wc = cover(Hin, Win, 10 ** 6, 10 ** 6, r)
        for H, W in ((hc, wc), (hc - 3, wc - 2), (hc + 5, wc + 4)):
            want, v, _ = mots_check(masks, list(range(6)), [1] * 6, thr, r, H, W, f"resize lattice {Hin}x{Win} r={r} {H}x{W}")
            assert v.shape[1:] == cover(Hin, Win, H, W, r)
            cmp += len(want)
            at_thr += int((v == thr32(thr)).sum())
    assert thr != 0.5 or at_thr > 0
    exact(cmp, f"mots resize lattice r={r} thr={thr} ({at_thr} pixels at thr)")


@gpu
def test_mots_encode_batched_64_images():
    """One uc_mots_encode_batched call over 64 images (UC_MOTS_MAX_IMAGES): every lattice ratio, frames covered, cropped and
    larger than the cover, k = 0 .. 6 instances with rows -1 and >= n_max, random emit; every image equals its own reference."""
    g, rg = G(64), rng(64)
    B, n_max, Hin, Win = 64, 6, 24, 20
    masks = torch.stack([blocky(n_max, Hin, Win, g, k=2) for _ in range(B)]).to(dev)
    ks, rs, Hs, Ws, order, emit, want = [], [], [], [], [], [], []
    for b in range(B):
        r = RATIOS[b % 4]
        hc, wc = cover(Hin, Win, 10 ** 6, 10 ** 6, r)
        H, W = [(hc, wc), (hc + 3, wc + 5), (max(1, hc - 4), wc - 1)][b % 3]
        k = b % 7
        o = rg.integers(-1, n_max + 2, k).tolist()
        e = rg.integers(0, 2, k).tolist()
        for lst, val in ((ks, k), (rs, r), (Hs, H), (Ws, W)):
            lst.append(val)
        order += o
        emit += e
        want.extend(mots_ref(masks[b], o, e, 0.5, r, H, W)[0])
    assert 0 in ks and any(o < 0 for o in order) and any(o >= n_max for o in order)
    K = len(order)
    cap = sum(map(len, want)) + 64
    ws = ops.mots_encode_workspace(K, max(Hs), max(Ws), dev)
    chars = torch.full((cap + 256,), SENT, dtype=torch.uint8, device=dev)
    offsets = torch.full((K + 1,), -1, dtype=torch.int64, device=dev)
    ops.mots_encode(masks, torch.tensor(order, dtype=torch.int32, device=dev), torch.tensor(emit, dtype=torch.uint8, device=dev), 0.5, rs,
                    Hs, Ws, ws, chars[:cap], offsets, k=ks)
    torch.cuda.synchronize()
    got, _ = strings_of(chars, offsets, K, cap)
    assert got == want
    exact(K, "mots batched B=64 (strings)")


@gpu
def test_mots_encode_capacity_clip():
    """Capacities 0, inside a multi-char count, at a string boundary, total - 1 and total: the prefix of the concatenated strings
    is written, the byte after the capacity keeps its sentinel, and the offsets are complete."""
    g = G(77)
    hm, wm = 401, 79
    c = delta_counts(hm * wm)
    bits = [bits_of(np.cumsum(c)[:-1], hm, wm), torch.rand(hm, wm, generator=g) < 0.3, torch.zeros(hm, wm, dtype=torch.bool)]
    masks = torch.stack([lattice(b, 0.5, g) for b in bits]).to(dev)
    order, emit = [0, 1, 2], [1, 1, 1]
    want, _, _ = mots_ref(masks, order, emit, 0.5, 1.0, hm, wm)
    full = "".join(want)
    T = len(full)
    inside = next(p for p in range(1, T) if (ord(full[p - 1]) - 48) & 0x20)  # the char before p continues a count
    caps = [0, inside, len(want[0]), T - 1, T]
    for cap in caps:
        ws = ops.mots_encode_workspace(3, hm, wm, dev)
        chars = torch.full((cap + 256,), SENT, dtype=torch.uint8, device=dev)
        offsets = torch.full((4,), -1, dtype=torch.int64, device=dev)
        ops.mots_encode(masks, torch.tensor(order, dtype=torch.int32, device=dev), torch.tensor(emit, dtype=torch.uint8, device=dev), 0.5,
                        1.0, hm, wm, ws, chars[:cap], offsets)
        torch.cuda.synchronize()
        assert offsets.cpu().tolist() == [0, len(want[0]), len(want[0]) + len(want[1]), T], cap
        assert bytes(chars[:cap].cpu().numpy()).decode("ascii") == full[:cap], cap
        assert bool((chars[cap:] == SENT).all()), f"capacity {cap}: chars past it were written"
    exact(len(caps) * (T + 4), f"mots capacity clip at {caps} of {T}")


# ================================================================================================ uc_vos_aggregate
def vos_masks(n, Hin, Win, tie, g):
    """n lattice masks with horizontal bands: tie[0] alone at 0.5 (background 0.5 ties it), tie[0:2] at 0.75, tie[0:3] at 0.75, all
    at 1.0 (saturated), every other mask 0 in those bands; random grid values elsewhere."""
    m = grid_values((n, Hin, Win), g)
    b = Hin // 6
    m[:, b:5 * b] = 0.0
    for j, (v, who) in enumerate(((0.5, tie[:1]), (0.75, tie[:2]), (0.75, tie[:3]))):
        for k in who:
            m[k, (1 + j) * b:(2 + j) * b] = v
    m[:, 4 * b:5 * b] = 1.0
    return m


def label_map(H, W, ids):
    lab = torch.zeros(H, W, dtype=torch.uint8)
    for j, oid in enumerate(ids):
        lab[5 * H // 6:, j * W // (len(ids) + 1):(j + 1) * W // (len(ids) + 1)] = oid
    return lab.to(dev)


@gpu
@pytest.mark.parametrize("r", RATIOS)
def test_vos_aggregate_lattice_ties(r):
    """uc_vos_aggregate on the lattice: soft masks and labels exactly equal, with the background tying one object at 0.5, two and
    three objects tying at 0.75 and at 1.0 with ids listed out of id order, initial-label-map objects between network masks (one id
    absent from the map), and frames covered exactly, cropped and larger than the cover (zeros beyond)."""
    g = G(int(100 * r))
    Hin, Win = 48, 40
    m = vos_masks(4, Hin, Win, [0, 1, 2], g).to(dev)
    hc, wc = cover(Hin, Win, 10 ** 6, 10 ** 6, r)
    videos = []
    for H, W in ((hc, wc), (hc - 5, wc - 3), (hc + 7, wc + 5)):
        lab = label_map(H, W, [4])
        objs = [(9, m[0], None), (3, m[1], None), (4, None, lab), (5, m[2], None), (200, None, lab), (1, m[3], None)]
        videos.append(dict(objs=objs, H=H, W=W, r=r, soft=True))
    assert any(cover(Hin, Win, v["H"], v["W"], r) < (v["H"], v["W"]) for v in videos)
    ties = vos_check(videos, Hin, Win, False, f"vos lattice r={r}")
    assert all(v > 0 for v in ties.values()), ties


@gpu
def test_vos_aggregate_object_counts_and_ids():
    """n = 1 (id 1, id 255) and n = 16 (kVosMaxObj) with ids 1 and 255 in a shuffled list, four of them from the label map (one id
    absent), ties among out-of-order ids, in a frame larger than the cover."""
    g = G(16)
    Hin, Win, r = 36, 24, 1.5
    hc, wc = cover(Hin, Win, 10 ** 6, 10 ** 6, r)
    H, W = hc + 4, wc + 3
    ids = [200, 17, 255, 1, 33, 90, 2, 128, 64, 5, 250, 7, 99, 3, 44, 11]
    m = vos_masks(12, Hin, Win, [0, 2, 1], g).to(dev)  # ties between ids 200, 255 and 17
    lab = label_map(H, W, [33, 7, 250])
    objs, j = [], 0
    for k, oid in enumerate(ids):
        if oid in (33, 7, 250, 11):  # 11 is absent from the label map
            objs.append((oid, None, lab))
        else:
            objs.append((oid, m[j], None))
            j += 1
    videos = [dict(objs=[(1, m[0], None)], H=H, W=W, r=r, soft=True), dict(objs=[(255, m[1], None)], H=H, W=W, r=r, soft=True),
              dict(objs=objs, H=H, W=W, r=r, soft=True)]
    ties = vos_check(videos, Hin, Win, False, "vos n=1 / n=16")
    assert all(v > 0 for v in ties.values()), ties


@gpu
def test_vos_aggregate_grid_stride_wraps():
    """A 1080 x 1920 frame: more pixels than the grid's threads (num_sms * 16 * 256), so the grid-stride loop wraps."""
    g = G(1080)
    Hin, Win = 540, 960
    assert 1080 * 1920 > torch.cuda.get_device_properties(0).multi_processor_count * 16 * 256
    m = vos_masks(3, Hin, Win, [2, 0, 1], g).to(dev)
    lab = label_map(1080, 1920, [6])
    objs = [(3, m[0], None), (1, m[1], None), (6, None, lab), (2, m[2], None)]
    ties = vos_check([dict(objs=objs, H=1080, W=1920, r=0.5, soft=True)], Hin, Win, False, "vos 1080x1920")
    assert all(v > 0 for v in ties.values()), ties


@gpu
def test_vos_aggregate_batched_64_videos():
    """uc_vos_aggregate_batched over 64 videos (UC_VOS_MAX_VIDEOS) with their own frame size, lattice ratio and 1 .. 16 objects
    (every fifth from a label map), soft outputs null for every third video; each video equals its own reference."""
    g, rg = G(6464), rng(6464)
    Hin, Win = 24, 20
    videos = []
    for b in range(64):
        r = RATIOS[b % 4]
        n = 1 + b % 16
        hc, wc = cover(Hin, Win, 10 ** 6, 10 ** 6, r)
        H, W = [(hc, wc), (hc + 3, wc + 2), (max(1, hc - 2), wc + 1)][b % 3]
        ids = rg.choice(np.arange(1, 256), n, replace=False).tolist()
        m = vos_masks(n, Hin, Win, list(rg.permutation(n)[:3]), g).to(dev)
        lab = label_map(H, W, ids[::5])
        objs = [(oid, None, lab) if k % 5 == 4 else (oid, m[k], None) for k, oid in enumerate(ids)]
        videos.append(dict(objs=objs, H=H, W=W, r=r, soft=b % 3 != 0))
    ties = vos_check(videos, Hin, Win, True, "vos batched B=64")
    assert all(v > 0 for v in ties.values()), ties


# ================================================================================================ uc_inst_encode_batched
def inst_images(hs, ws, f, n_max, row0):
    """Images of one instance encode: every lattice ratio, H % 32 in {0, 1, 31}, frames cropped, exact and larger than the cover,
    and counts whose window of n_max rows from row0 is full, partial, empty or negative (count < row0)."""
    Hin, Win = hs * f, ws * f
    imgs = []
    counts = [row0 + n_max + 2, row0 + 2, row0, max(row0 - 2, 0), row0 + n_max, row0 + 1, 0, row0 + 3]
    for b in range(8):
        r = RATIOS[b % 4]
        hc, wc = cover(Hin, Win, 10 ** 6, 10 ** 6, r)
        H = [32 * (hc // 32 + 1), 32 * (hc // 32) + 1, 32 * (hc // 32) + 31, hc][(b // 2) % 4]
        W = [wc, wc + 3, max(1, wc - 2)][b % 3]
        imgs.append((r, H, W, counts[b]))
    return imgs


@gpu
@pytest.mark.parametrize("thr", THRS)
@pytest.mark.parametrize("f", FACTORS)
def test_inst_encode_lattice(f, thr):
    """uc_inst_encode_batched on the lattice, every (image, row) slot against aligned_bilinear (x f, float64) + resize + threshold
    over the whole H x W frame (background beyond the cover), at row0 = 0 and 5; the emit flags equal count - row0 > row."""
    hs, ws, n_max = 12, 10, 4
    cmp, at_thr, hmod, short = 0, 0, set(), 0
    for row0 in (0, 5):
        g = G(100 * f + row0)
        imgs = inst_images(hs, ws, f, n_max, row0)
        B = len(imgs)
        maps = torch.stack([blocky(n_max, hs, ws, g, k=2) for _ in range(B)])
        rs, Hs, Ws, counts = (list(t) for t in zip(*imgs))
        want, emit_ref = [], []
        for b, (r, H, W, count) in enumerate(imgs):
            up = ab_upsample(maps[b], f)
            v = resize64(up, r, H, W)
            at_thr += int((v == thr32(thr)).sum())
            hmod.add(H % 32)
            short += v.shape[1] < H or v.shape[2] < W
            for i in range(n_max):
                on = i < count - row0
                emit_ref.append(int(on))
                frame = np.zeros((H, W), dtype=bool)
                frame[:v.shape[1], :v.shape[2]] = (v[i] > thr32(thr)).numpy()
                want.append(R.rle_encode(frame) if on else "")
        got, emit = inst_run(maps.to(dev), counts, row0, f, thr, rs, Hs, Ws, sum(map(len, want)) + 64)
        assert emit == emit_ref
        assert got == want, f"first differing slot {next(i for i in range(len(want)) if got[i] != want[i])}"
        assert set(emit_ref) == {0, 1} and any(c < row0 for c in counts) == (row0 > 0)
        cmp += len(want) + len(emit)
    assert {0, 1, 31} <= hmod and short > 0 and (thr != 0.5 or at_thr > 0), (hmod, short, at_thr)
    exact(cmp, f"inst lattice f={f} thr={thr} (strings + emit; {at_thr} pixels at thr)")


def dyn_maps(h, w, level_hw, up, f, n_max, seed):
    """The d_rate = 1 maps and the d_rate = f stored masks of uc_dynamic_masks for the same instances (test_sampling_edges_gpu's
    inputs: tied, saturated and random convex weights, edge anchors)."""
    g = G(seed)
    feats, um, dyn = mask_case(h, w, level_hw, up, 169, g)
    ws = ops.PostWorkspace(sum(a * b for a, b in level_hw), dev)
    ws.anchors[:n_max] = torch.tensor(edge_anchors(level_hw, g, n_max), dtype=torch.int32, device=dev)
    ws.count.fill_(n_max)
    maps = ops.dynamic_masks(feats, um, dyn, level_hw, ws, n_max, up_rate=up, d_rate=1).clone()
    stored = ops.dynamic_masks(feats, um, dyn, level_hw, ws, n_max, up_rate=up, d_rate=f).clone()
    torch.cuda.synchronize()
    return maps, stored


def pick_thresholds(vals, exact_vals, rg, per):
    """`per` values of each map taken at pixels in (0.02, 0.98) where rounding happened (the value differs from the exact one),
    each with the float just below it."""
    out = []
    for i in range(vals.shape[0]):
        v, e = vals[i].reshape(-1), exact_vals[i].reshape(-1)
        idx = torch.nonzero((v > 0.02) & (v < 0.98) & (v.double() != e)).flatten()
        assert idx.numel() >= per, "too few rounded pixels"
        for j in rg.choice(idx.numel(), per, replace=False):
            t = v[idx[int(j)]]
            out += [float(t), float(torch.nextafter(t, torch.tensor(0.0)))]
    return out


@gpu
@pytest.mark.parametrize("f", (2, 3, 4))
def test_inst_encode_rounding_order_pin(f):
    """r = 1: the fused bit of every pixel is exactly stored > thr, stored the uc_dynamic_masks output at d_rate = f for the same
    instances, at thresholds equal to stored values (and one float below) at pixels where the upsample rounds.  f = 3 takes the
    division path of ab_coord.  stored itself equals the float32 emulation of the documented order."""
    (h, w), level_hw = MASK_MAPS[1]
    up, n_max = 4, 6
    maps, stored = dyn_maps(h, w, level_hw, up, f, n_max, 7000 + f)
    s_cpu = stored.cpu()
    assert torch.equal(final_up_emul(maps.cpu(), f), s_cpu), "mask_final_up_kernel is not fma(1 - fy, top, fy bot) of fma rows"
    H, W = stored.shape[1:]
    cmp, at_thr = 0, 0
    for thr in pick_thresholds(s_cpu, ab_upsample(maps.cpu(), f), rng(f), 4):
        got, emit = inst_run(maps[None], [n_max], 0, f, thr, [1.0], [H], [W], 1 << 20)
        bits = (s_cpu > np.float32(thr)).numpy()
        assert got == [R.rle_encode(bits[i]) for i in range(n_max)], f"thr {thr!r}"
        assert emit == [1] * n_max
        at_thr += int((s_cpu == np.float32(thr)).sum())
        cmp += n_max * H * W
    assert at_thr > 0
    exact(cmp, f"inst rounding pin f={f} (pixel bits; {at_thr} pixels exactly at thr)")


ROUND_CASES = [(4, 800 / 402, (50, 5), [(50, 5), (25, 3), (13, 2)], 402, 41), (3, 1.5, MASK_MAPS[1][0], MASK_MAPS[1][1], 110, 160),
               (2, 0.5, MASK_MAPS[1][0], MASK_MAPS[1][1], 200, 340)]


@gpu
@pytest.mark.parametrize("f,r,hw,level_hw,H,W", ROUND_CASES)
def test_inst_encode_equals_mots_encode_off_lattice(f, r, hw, level_hw, H, W):
    """r != 1 (800 / 402: one row short of the frame): the fused strings equal uc_mots_encode of the stored d_rate = f masks, padded
    to the H x W frame, at thresholds taken from the float32 emulation of resize_mix on the emulated upsample; the stored masks'
    resize (mots_planes_kernel) equals that emulation bit for bit."""
    h, w = hw
    up, n_max = 4, 4
    maps, stored = dyn_maps(h, w, level_hw, up, f, n_max, 7100 + f)
    s_cpu = stored.cpu()
    assert torch.equal(final_up_emul(maps.cpu(), f), s_cpu)
    Hin, Win = stored.shape[1:]
    hm, wm = cover(Hin, Win, H, W, r)
    assert (hm, wm) != (H, W)
    emul = resize_emul(s_cpu, r, H, W)
    cmp, at_thr = 0, 0
    for thr in pick_thresholds(emul, resize64(s_cpu, r, H, W), rng(f + 10), 3):
        got, emit = inst_run(maps[None], [n_max], 0, f, thr, [r], [H], [W], 1 << 20)
        assert emit == [1] * n_max
        for i in range(n_max):
            s, _ = mots_run(stored, [i], [1], thr, r, H, W, 1 << 20)
            frame = np.zeros((H, W), dtype=bool)
            frame[:hm, :wm] = R.rle_decode(s[0], hm, wm)
            assert np.array_equal(frame[:hm, :wm], (emul[i] > np.float32(thr)).numpy()), f"mots slot {i} thr {thr!r} vs the emulation"
            assert got[i] == R.rle_encode(frame), f"slot {i} thr {thr!r}"
        at_thr += int((emul == np.float32(thr)).sum())
        cmp += n_max
    exact(cmp, f"inst vs mots r={r:.4f} f={f} (strings; {at_thr} emulated pixels at thr)")

"""The oracle's emulation of torchvision's IoU arithmetic, off the GPU: fma32 (fmaf in numpy) against exact rational arithmetic on
random and midpoint triples, box_iou_f32 against torchvision.ops.box_iou, and the near-threshold pairs the NMS edge tests
(tests/test_post_edges_gpu.py) are built from, where fusing one area or the other, or none, decides differently."""
import math
import os
import sys
from fractions import Fraction

import numpy as np
import pytest
import torch
import torchvision

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import unicorn_oracle as orc  # noqa: E402

f32 = np.float32
GRID = 2.0 ** -11  # below 4096, (x1 + x2) / 2 and x2 - x1 of grid values are exact in float32


def round_f32(x):
    """A Fraction rounded to the nearest float32, ties to even (normal and subnormal range)."""
    if x == 0:
        return 0.0
    s, x = (-1 if x < 0 else 1), abs(x)
    e = x.numerator.bit_length() - x.denominator.bit_length()
    if x < Fraction(2) ** e:
        e -= 1
    e = max(e, -126)
    return s * math.ldexp(round(x / Fraction(2) ** (e - 23)), e - 23)


def exact_fma(a, b, c):
    return np.array([round_f32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))) for x, y, z in zip(a, b, c)], f32)


def midpoint_triples(n, rng):
    """a * b = +-(1 - 2^-46) 2^k and c an odd or even multiple of 2^(k+1) in [2^(k+24), 2^(k+25)): the float64 sum is the
    float32 midpoint c +- 2^k, and the exact sum lies 2^(k-46) to one side of it."""
    k = rng.integers(-40, 40, n)
    sa, sb, sc = (rng.choice([-1.0, 1.0], n) for _ in range(3))
    a = (sa * (1 + 2.0 ** -23) * np.exp2(k // 2)).astype(f32)
    b = (sb * (1 - 2.0 ** -23) * np.exp2(k - k // 2)).astype(f32)
    c = (sc * rng.integers(2 ** 23, 2 ** 24, n) * np.exp2(k + 1.0)).astype(f32)
    return a, b, c


def test_fma32_matches_exact_rounding():
    rng = np.random.default_rng(0)
    n = 20000
    a = (rng.uniform(-1, 1, n) * np.exp2(rng.integers(-30, 30, n))).astype(f32)
    b = (rng.uniform(-1, 1, n) * np.exp2(rng.integers(-30, 30, n))).astype(f32)
    c = (rng.uniform(-1, 1, n) * np.exp2(rng.integers(-60, 60, n))).astype(f32)
    c[: n // 4] = -(a[: n // 4].astype(np.float64) * b[: n // 4]).astype(f32)  # cancellation: the result is the product's tail
    assert np.array_equal(orc.fma32(a, b, c), exact_fma(a, b, c))
    ma, mb, mc = midpoint_triples(4000, rng)
    want = exact_fma(ma, mb, mc)
    naive = (ma.astype(np.float64) * mb + mc).astype(f32)  # float64 then float32: a second rounding at the midpoint
    assert (naive != want).sum() > 1000
    assert np.array_equal(orc.fma32(ma, mb, mc), want)
    # box-like operands: widths and heights on the coordinate grid and an area
    w, h = (np.round(rng.uniform(1, 300, (2, n)) / GRID) * GRID).astype(f32)
    s = (w * h)[::-1].copy()
    assert np.array_equal(orc.fma32(w, h, s), exact_fma(w, h, s))
    print(f"exact: {n} random, {n} cancelling, 4000 midpoint ({(naive != want).sum()} double-rounded in float64), {n} box triples")


def test_box_iou_f32_matches_torchvision_box_iou():
    rng = np.random.default_rng(1)
    a = (np.round(rng.uniform(0, 300, (200, 4)) / GRID) * GRID).astype(f32)
    b = (np.round(rng.uniform(0, 300, (150, 4)) / GRID) * GRID).astype(f32)
    a[:, 2:] += a[:, :2]
    b[:, 2:] += b[:, :2]
    tv = torchvision.ops.box_iou(torch.from_numpy(a), torch.from_numpy(b)).numpy()
    emu = orc.box_iou_f32(a, b)
    assert np.array_equal(emu.view(np.int32), tv.view(np.int32)) and (tv > 0).sum() > 5000
    print(f"exact: {tv.size} IoUs")


def conventions(a, b):
    """IoU of earlier box a and later box b with b's area fused (devIoU), a's area fused, and nothing fused."""
    w = np.maximum(np.minimum(a[..., 2], b[..., 2]) - np.maximum(a[..., 0], b[..., 0]), f32(0))
    h = np.maximum(np.minimum(a[..., 3], b[..., 3]) - np.maximum(a[..., 1], b[..., 1]), f32(0))
    inter = w * h
    wa, ha, wb, hb = a[..., 2] - a[..., 0], a[..., 3] - a[..., 1], b[..., 2] - b[..., 0], b[..., 3] - b[..., 1]
    sa, sb = wa * ha, wb * hb
    return (inter / (orc.fma32(wb, hb, sa) - inter), inter / (orc.fma32(wa, ha, sb) - inter), inter / ((sa + sb) - inter))


def near_pairs(thr, n, seed, K=48):
    """n <= 256 box pairs (a, b), one per 240-pixel cell of a 16 x 16 grid (pairs never overlap each other), on the exact
    coordinate grid, each with IoU within a few ulps of float32(thr).  Pair i is of kind ("flip", "eq", "ulp+", "ulp-")[i % 4]
    where the scan finds one: "flip" decides differently with a's area fused or with nothing fused than with b's (devIoU),
    "eq" has devIoU == float32(thr), "ulp+" / "ulp-" one ulp above / below; otherwise the pair nearest the threshold ("near").
    b is a shifted right by about the IoU-thr offset and its bottom edge moved, over a (2K)^2 grid of GRID steps."""
    assert n <= 256
    rng = np.random.default_rng(seed)
    T = f32(thr)
    i = np.arange(n)
    snap = lambda v: np.round(v / GRID) * GRID  # noqa: E731
    x1, y1 = (i % 16) * 240.0 + snap(rng.uniform(0, 20, n)), (i // 16) * 240.0 + snap(rng.uniform(0, 20, n))
    wa, ha = snap(rng.uniform(30, 100, n)), snap(rng.uniform(30, 100, n))
    a = np.stack([x1, y1, x1 + wa, y1 + ha], 1).astype(f32)
    d = np.arange(-K, K) * GRID
    sx = snap(wa * (1 - thr) / (1 + thr))[:, None] + np.repeat(d, 2 * K)[None]
    b = np.repeat(a[:, None, :].astype(np.float64), (2 * K) ** 2, 1)
    b[..., 0] += sx
    b[..., 2] += sx
    b[..., 3] += np.tile(d, 2 * K)[None]
    b = b.astype(f32)
    fb, fa, un = conventions(np.repeat(a[:, None, :], (2 * K) ** 2, 1), b)
    cats = [((fb > T) != (fa > T)) | ((fb > T) != (un > T)), fb == T, fb == np.nextafter(T, f32(1)), fb == np.nextafter(T, f32(0))]
    names = np.array(["flip", "eq", "ulp+", "ulp-"])
    pick = np.abs(fb.astype(np.float64) - float(T)).argmin(1)
    kind = np.full(n, "near", dtype=object)
    for r in range(n):
        for c in [r % 4] + [c for c in range(4) if c != r % 4]:
            if cats[c][r].any():
                pick[r], kind[r] = cats[c][r].argmax(), names[c]
                break
    return a, b[i, pick], kind.astype(str)


@pytest.mark.parametrize("thr", (0.3, 0.5, 0.6, 0.65, 0.7))
def test_near_pairs_separate_the_conventions(thr):
    a, b, kind = near_pairs(thr, 256, seed=11)
    T = f32(thr)
    fb, fa, un = conventions(a, b)
    assert np.array_equal(orc.dev_iou(a, b), fb)
    flip = kind == "flip"
    assert flip.sum() >= 10 and ((fb[flip] > T) != (fa[flip] > T)).sum() >= 5 and ((fb[flip] > T) != (un[flip] > T)).sum() >= 5
    assert (fb[kind == "eq"] == T).sum() >= 20
    assert (fb[kind == "ulp+"] == np.nextafter(T, f32(1))).sum() >= 20 and (fb[kind == "ulp-"] == np.nextafter(T, f32(0))).sum() >= 20
    assert a.max() < 4096 and b.max() < 4096 and (b[:, 2] > b[:, 0]).all()
    print(f"thr {thr}: {dict(zip(*np.unique(kind, return_counts=True)))}")

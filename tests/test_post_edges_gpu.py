"""Detection post-processing (csrc/post.cu) and uc_box_iou (csrc/assoc.cu) against torchvision's arithmetic at the edges where
a decision flips: near-threshold IoU pairs in both NMS stages, suppression chains across the 64-bit words and 256-candidate
chunks, a kept list spilling out of shared memory, candidate counts around powers of two and the 65536-key sort, equal scores,
max_keep prefixes, classes, batches with different counts, the score filter at conf, and the decode against float64.

Every NMS result is compared exactly (rows bit for bit, order, count, anchors) with torchvision.ops.nms on CUDA, run one class
at a time, merged in descending score and ascending candidate index; where scores tie, with the stable greedy emulation of the
oracle (unicorn_oracle.nms_greedy on its devIoU emulation).  torchvision's batched_nms offsets the boxes of each class by a
per-class constant on CUDA up to 5000 boxes, which re-rounds every IoU; that path is not a reference here.

Boxes are built on a 2^-11 grid below 4096, where cx = (x1 + x2) / 2 and w = x2 - x1 are exact, so the corners the filter
computes from (cx, cy, w, h) are the boxes themselves.  Every check prints its count of exact comparisons or its err/bound."""
import os
import sys

import numpy as np
import pytest
import torch
import torchvision

from unicorn_b200 import ops, post_ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import unicorn_oracle as orc  # noqa: E402
from test_post_oracle import near_pairs  # noqa: E402

pytestmark = pytest.mark.gpu
dev = "cuda"
f32 = np.float32
THRS = (0.3, 0.5, 0.6, 0.65, 0.7)


# ----------------------------------------------------------------------------------------------- inputs and references
def pred_of(boxes, scores, cls=None, ncls=1):
    """Decoded head rows [A, 5 + ncls] (cx, cy, w, h, obj, class probabilities) whose candidates are exactly `boxes` with
    score obj * 1.0 = `scores` and class `cls` (other classes 0.5)."""
    boxes = np.asarray(boxes, dtype=np.float64)
    A = boxes.shape[0]
    p = np.zeros((A, 5 + ncls), dtype=np.float32)
    p[:, 0] = (boxes[:, 0] + boxes[:, 2]) / 2
    p[:, 1] = (boxes[:, 1] + boxes[:, 3]) / 2
    p[:, 2] = boxes[:, 2] - boxes[:, 0]
    p[:, 3] = boxes[:, 3] - boxes[:, 1]
    p[:, 4] = scores
    p[:, 5:] = 0.5
    p[np.arange(A), 5 + (np.zeros(A, dtype=np.int64) if cls is None else np.asarray(cls))] = 1.0
    t = torch.from_numpy(p)
    assert np.array_equal(corners(t).numpy(), boxes.astype(np.float32)), "boxes off the exact grid"
    assert np.array_equal(p[:, 4].astype(np.float64), np.asarray(scores, dtype=np.float64)), "scores not float32"
    return t


def corners(p):
    return torch.stack([p[:, 0] - p[:, 2] / 2, p[:, 1] - p[:, 3] / 2, p[:, 0] + p[:, 2] / 2, p[:, 1] + p[:, 3] / 2], 1)


def candidates(p, ncls, conf):
    """The filter of postprocess (utils/boxes.py): det rows and anchor ids of the anchors with rn(obj * class_conf) >= conf,
    class_conf / class_pred the first maximum."""
    cls = p[:, 5:5 + ncls].numpy()
    cp = torch.from_numpy(np.argmax(cls, 1))
    cc = p[torch.arange(p.shape[0]), 5 + cp]
    mask = p[:, 4] * cc >= np.float32(conf)
    det = torch.cat([corners(p), p[:, 4:5], cc[:, None], cp[:, None].float()], 1)[mask]
    return det, torch.nonzero(mask)[:, 0]


def reference(p, ncls, conf, thr, agnostic=False, stable=False):
    """postprocess of one image: rows [n, 7] and anchors [n].  stable=False: torchvision.ops.nms on CUDA per class;
    stable=True: the oracle's greedy emulation (equal scores in ascending candidate index)."""
    det, anc = candidates(p, ncls, conf)
    scores = det[:, 4] * det[:, 5]
    groups = [np.arange(det.shape[0])] if agnostic else [np.nonzero(det[:, 6].numpy() == c)[0] for c in np.unique(det[:, 6].numpy())]
    keep = []
    for idx in groups:
        if len(idx) == 0:
            continue
        if stable:
            k = orc.nms_greedy(det[idx, :4].numpy(), scores[idx].numpy(), thr)
        else:
            k = torchvision.ops.nms(det[idx, :4].to(dev), scores[idx].to(dev), thr).cpu().numpy()
        keep.append(idx[k])
    keep = np.sort(np.concatenate(keep)) if keep else np.zeros(0, dtype=np.int64)
    keep = keep[np.argsort(-scores[keep].numpy(), kind="stable")]
    return det[keep], anc[keep]


def run(p, ncls, conf, thr, max_keep=0, agnostic=False):
    """uc_postprocess_batched_ex on one image: rows [n, 7] and anchors [n] on the host."""
    ws = ops.PostWorkspace(p.shape[0], dev)
    post_ops.postprocess_device_ex(p.to(dev).contiguous(), ncls, conf, thr, ws, max_keep=max_keep, class_agnostic=agnostic)
    n = int(ws.count[0].item())
    return ws.dets[:n].cpu(), ws.anchors[:n].cpu()


def same(got, ref, name):
    (d, a), (rd, ra) = got, ref
    assert d.shape[0] == rd.shape[0], f"{name}: {d.shape[0]} rows kept, reference {rd.shape[0]}"
    assert torch.equal(a, ra.to(a.dtype)), f"{name}: anchors differ at rows {torch.nonzero(a != ra.to(a.dtype))[:8, 0].tolist()}"
    assert torch.equal(d.view(torch.int32), rd.contiguous().view(torch.int32)), f"{name}: rows differ"
    print(f"exact: {d.shape[0]} rows  {name}")
    return d.shape[0]


def disjoint(n, size=40, pitch=60, seed=0):
    """n pairwise disjoint boxes on integer coordinates, row by row in a 64-wide grid of cells."""
    i = np.arange(n)
    x, y = (i % 64) * pitch, (i // 64) * pitch
    assert y.max(initial=0) + pitch < 4096
    return np.stack([x, y, x + size, y + size], 1).astype(f32)


def ranked(n, offset=0):
    """n distinct float32 scores in descending order, exact multiples of 2^-18."""
    return ((2 ** 18 - 1 - offset - np.arange(n)) * 2.0 ** -18).astype(f32)


def random_boxes(n, rng, span=1200.0):
    """n boxes on the exact grid, clustered so that NMS suppresses a good share of them."""
    q = 2.0 ** -11
    k = rng.integers(0, max(1, n // 12), n)
    c = rng.uniform(100, span, (max(1, n // 12), 2))[k] + rng.normal(0, 6, (n, 2))
    wh = rng.uniform(20, 120, (max(1, n // 12), 2))[k] * rng.uniform(0.85, 1.15, (n, 2))
    b = np.concatenate([c - wh / 2, c + wh / 2], 1)
    return (np.round(np.clip(b, 0, 4000) / q) * q).astype(f32)


# ----------------------------------------------------------------------------------------------- near-threshold IoU
@pytest.mark.parametrize("thr", THRS)
def test_dev_iou_emulation_matches_torchvision_nms(thr):
    """The oracle's devIoU decides every constructed pair as torchvision.ops.nms on CUDA does, and the pairs include ones where
    fusing the other box's area, or fusing nothing, would decide differently."""
    a, b, kind = near_pairs(thr, 256, seed=11)
    n = a.shape[0]
    boxes = torch.from_numpy(np.concatenate([a, b]))
    scores = torch.from_numpy(np.concatenate([np.full(n, 0.9, f32), np.full(n, 0.5, f32)]))
    keep = torchvision.ops.nms(boxes.to(dev), scores.to(dev), thr).cpu().numpy()
    tv_sup = ~np.isin(np.arange(n, 2 * n), keep)
    assert np.isin(np.arange(n), keep).all()  # the pairs are in disjoint cells: every first box is kept
    emu = orc.dev_iou(a, b) > f32(thr)
    assert np.array_equal(tv_sup, emu), f"{(tv_sup != emu).sum()} of {n} pairs decided differently from torchvision"
    print(f"exact: {n} pair decisions at thr {thr}: {dict(zip(*np.unique(kind, return_counts=True)))}, {emu.sum()} suppressed")


@pytest.mark.parametrize("thr", THRS)
@pytest.mark.parametrize("stage", [1, 2])
def test_near_threshold_pairs(stage, thr):
    """Stage 1: every first box is in chunk 0 and every second box in chunk 1 (tested against the kept list); stage 2: each
    pair is adjacent in one chunk (tested pairwise).  IoUs equal to float32(thr), one ulp either side, and pairs where the
    fused operand decides, at positions 0..511."""
    a, b, kind = near_pairs(thr, 256, seed=int(thr * 100) + stage)
    n = a.shape[0]
    assert n == 256
    if stage == 1:
        boxes, order = np.concatenate([a, b]), np.arange(2 * n)
    else:
        boxes = np.stack([a, b], 1).reshape(2 * n, 4)
        order = np.arange(2 * n)
    scores = ranked(2 * n)[order]
    perm = np.random.default_rng(stage).permutation(2 * n)  # anchors in a scrambled order: the sort puts them back
    p = pred_of(boxes[perm], scores[perm])
    got = run(p, 1, 0.01, thr)
    same(got, reference(p, 1, 0.01, thr), f"stage {stage} thr {thr}")
    same(got, reference(p, 1, 0.01, thr, stable=True), f"stage {stage} thr {thr} vs emulation")
    sup = 2 * n - got[0].shape[0]
    assert 0 < sup < n, sup
    print(f"  {sup} second boxes suppressed; kinds {dict(zip(*np.unique(kind, return_counts=True)))}")


# ----------------------------------------------------------------------------------------------- chains, spill, counts
def chain(n, x0=0.0, y0=0.0):
    """n boxes 10 wide shifted by 2: IoU(i, i+1) = 2/3 and IoU(i, i+2) = 3/7 at thr 0.5, so greedy keeps every other box and a
    suppressed box does not suppress its successor."""
    i = np.arange(n)
    x = x0 + 2.0 * (i % 1500)
    y = y0 + 20.0 * (i // 1500)
    return np.stack([x, y, x + 10, y + 10], 1).astype(f32)


@pytest.mark.parametrize("lead", [0, 1, 62, 63, 127, 191, 255])
def test_suppression_chains_across_words_and_chunks(lead):
    """`lead` isolated boxes, then one chain of 700 boxes in score order: it crosses candidate positions 63/64, 127/128,
    191/192, 255/256 and 511/512 with both parities of kept boxes."""
    iso = disjoint(lead) + np.array([0, 3000, 0, 3000], f32) if lead else np.zeros((0, 4), f32)
    boxes = np.concatenate([iso, chain(700)])
    p = pred_of(boxes, ranked(len(boxes)))
    got = run(p, 1, 0.01, 0.5)
    n = same(got, reference(p, 1, 0.01, 0.5), f"chain after {lead} boxes")
    assert n == lead + 350


def test_kept_list_spills_past_shared_memory():
    """3328 disjoint boxes are kept (indices past kNmsKeepSmem = 3072 live in the output rows), then candidates in later chunks
    that only one kept box suppresses: kept indices 0, 3071, 3072, 3073, 3100, 3327."""
    K = 3328
    kept = disjoint(K)
    targets = np.array([0, 3071, 3072, 3073, 3100, 3327])
    dup = kept[targets] + np.array([1, 0, 1, 0], f32)  # IoU 39/41 with its target only
    free = disjoint(4096)[K:K + 10]  # boxes of no one
    boxes = np.concatenate([kept, dup, free])
    scores = ranked(len(boxes))
    p = pred_of(boxes, scores)
    got = run(p, 1, 0.01, 0.5)
    n = same(got, reference(p, 1, 0.01, 0.5), "spilled kept list")
    assert n == K + 10 and n > 3072
    # class-aware with two classes: the targets' duplicates of the other class survive
    cls = np.zeros(len(boxes), dtype=np.int64)
    cls[K:K + 3] = 1
    p2 = pred_of(boxes, scores, cls, ncls=2)
    got2 = run(p2, 2, 0.01, 0.5)
    assert same(got2, reference(p2, 2, 0.01, 0.5), "spilled kept list, two classes") == K + 13
    for mk in (1, 255, 256, 257, 3071, 3072, 3073, 3074):
        part = run(p, 1, 0.01, 0.5, max_keep=mk)
        assert part[0].shape[0] == mk and torch.equal(part[0], got[0][:mk]) and torch.equal(part[1], got[1][:mk]), mk
    print("exact: max_keep 1, 255-257, 3071-3074 are prefixes of the full result")


@pytest.mark.parametrize("n", [0, 1, 63, 64, 65, 255, 256, 257, 512, 1023, 1024, 1025, 2048, 4096, 8192])
def test_candidate_counts(n):
    """n of 8192 anchors pass the filter, at scattered anchors; the rest score below conf."""
    rng = np.random.default_rng(n)
    A = 8192
    boxes = random_boxes(A, rng)
    scores = np.full(A, 0.005, f32)
    pick = rng.choice(A, n, replace=False)
    scores[pick] = ranked(n)[rng.permutation(n)] if n else scores[pick]
    p = pred_of(boxes, scores)
    got = run(p, 1, 0.01, 0.65)
    k = same(got, reference(p, 1, 0.01, 0.65), f"{n} of {A} candidates")
    assert (k == 0) == (n == 0)


@pytest.mark.parametrize("A", [21000, 64512])
def test_full_size_all_anchors_pass(A):
    """Every anchor of an 800x1280 (21000) or 1536x2048 (64512: a 65536-key sort) frame is a candidate."""
    rng = np.random.default_rng(A)
    boxes = random_boxes(A, rng, span=3800.0)
    p = pred_of(boxes, ranked(A)[rng.permutation(A)])
    got = run(p, 1, 0.0, 0.65)
    k = same(got, reference(p, 1, 0.0, 0.65), f"all {A} anchors pass")
    assert 0 < k < A


def test_equal_scores_keep_ascending_candidate_order():
    """Scores from a set of four values: the kept rows are in descending score and, within a score, ascending anchor; greedy
    visits equal scores in that order (against the stable emulation: torchvision does not promise an order for ties)."""
    rng = np.random.default_rng(5)
    A = 3000
    boxes = random_boxes(A, rng, span=900.0)
    scores = np.array([0.25, 0.5, 0.625, 0.75], f32)[rng.integers(0, 4, A)]
    p = pred_of(boxes, scores)
    for thr in (0.3, 0.65):
        got = run(p, 1, 0.01, thr)
        same(got, reference(p, 1, 0.01, thr, stable=True), f"tied scores thr {thr}")
        a, s = got[1].numpy(), got[0][:, 4].numpy()
        assert all(s[i] > s[i + 1] or (s[i] == s[i + 1] and a[i] < a[i + 1]) for i in range(len(a) - 1))
    q = pred_of(disjoint(A), scores)  # nothing suppressed: the output is the stable sort itself
    got = run(q, 1, 0.01, 0.5)
    assert torch.equal(got[1], torch.from_numpy(np.argsort(-scores, kind="stable")).int())
    print(f"exact: {A} tied-score rows in stable order")


@pytest.mark.parametrize("ncls", [1, 8, 80])
def test_classes(ncls):
    """Class-aware NMS per class and class-agnostic NMS over all, against torchvision; a box duplicated with another class is
    kept twice when class-aware and once when agnostic."""
    rng = np.random.default_rng(ncls)
    A = 4000
    boxes = random_boxes(A, rng)
    boxes[1] = boxes[0]
    cls = rng.integers(0, ncls, A)
    cls[1] = (cls[0] + 1) % ncls
    scores = ranked(A)
    p = pred_of(boxes, scores, cls, ncls)
    for agn in (False, True):
        got = run(p, ncls, 0.01, 0.65, agnostic=agn)
        same(got, reference(p, ncls, 0.01, 0.65, agnostic=agn), f"ncls {ncls} {'agnostic' if agn else 'class-aware'}")
        twice = int(np.isin([0, 1], got[1].numpy()).sum())
        assert twice == (1 if agn or ncls == 1 else 2), twice
    # random class probabilities: scores are rounded products and the class is an argmax
    p[:, 5:] = torch.from_numpy(rng.uniform(0, 1, (A, ncls)).astype(f32))
    p[:, 4] = torch.from_numpy(rng.uniform(0, 1, A).astype(f32))
    det, _ = candidates(p, ncls, 0.01)
    s = (det[:, 4] * det[:, 5]).numpy()
    stable = len(np.unique(s)) < len(s)
    for agn in (False, True):
        same(run(p, ncls, 0.01, 0.65, agnostic=agn), reference(p, ncls, 0.01, 0.65, agnostic=agn, stable=stable),
             f"ncls {ncls} random probabilities {'agnostic' if agn else 'class-aware'}")


def test_score_filter_at_conf():
    """obj * class_conf rounded to float32 and compared >= conf: products exactly at float32(conf), one ulp below and above, and
    rounded products around it; class_conf is the first maximum of equal class probabilities."""
    rng = np.random.default_rng(9)
    conf = 0.01
    c = np.float32(conf)
    n = 2000
    obj = rng.uniform(0.011, 0.9, n).astype(f32)
    best = (c / obj).astype(f32)
    best = np.nextafter(best, np.where(rng.integers(0, 2, n) > 0, 2, 0).astype(f32))  # products within an ulp or two of conf
    obj[:3], best[:3] = [c, np.nextafter(c, f32(0)), np.nextafter(c, f32(1))], 1.0
    ncls = 8
    p = pred_of(disjoint(n), obj, ncls=ncls)
    cls = rng.uniform(0, 1, (n, ncls)).astype(f32)
    cls[np.arange(n), rng.integers(0, ncls, n)] = best
    cls[np.arange(n), rng.integers(0, ncls, n)] = best  # often a second class with the same probability
    p[:, 5:] = torch.from_numpy(np.minimum(cls, best[:, None]))
    prod = torch.from_numpy(obj) * torch.from_numpy(best)
    npass = int((prod >= c).sum())
    assert 100 < npass < n - 100 and prod[0] == c and prod[1] < c
    ties = int(((p[:, 5:] == torch.from_numpy(best)[:, None]).sum(1) > 1).sum())
    assert ties > 100
    got = run(p, ncls, conf, 0.5)
    same(got, reference(p, ncls, conf, 0.5, stable=True), f"score filter at conf, {npass} of {n} pass, {ties} tied class maxima")
    assert set(got[1].tolist()) == set(torch.nonzero(prod >= c)[:, 0].tolist()) and 0 in got[1].tolist() and 1 not in got[1].tolist()


# ----------------------------------------------------------------------------------------------- batches
def _maps(B, hw, ncls, counts, rng):
    """Raw head maps (NHWC fp32 per level) whose image b has counts[b] anchors with obj logit 4, the rest -20."""
    A = sum(h * w for h, w in hw)
    ro, cl = [], []
    obj = np.full((B, A), -20.0, f32)
    logit = rng.normal(0, 2, (B, A, ncls)).astype(f32)
    for b, n in enumerate(counts):
        pick = rng.choice(A, n, replace=False)
        obj[b, pick] = rng.uniform(0, 4, n)
        logit[b, pick, rng.integers(0, ncls, n)] = 3.0  # score >= sigmoid(0) * sigmoid(3) > conf
    s = 0
    for h, w in hw:
        r = rng.normal(0, 0.5, (B, h, w, 5)).astype(f32)
        r[..., 4] = obj[:, s:s + h * w].reshape(B, h, w)
        ro.append(torch.from_numpy(r).to(dev))
        cl.append(torch.from_numpy(logit[:, s:s + h * w].reshape(B, h, w, ncls)).to(dev))
        s += h * w
    return ro, cl


@pytest.mark.parametrize("B", [1, 2, 3, 4])
@pytest.mark.parametrize("ncls", [1, 8])
def test_batched_images_with_different_counts(B, ncls):
    """uc_postprocess_batched_ex on decoded rows and uc_det_candidates_batched + uc_postprocess_nms_batched on the head maps,
    each image against its own reference; one image of each batch (the second, or the only one) has no candidate."""
    from unicorn_b200.engine import STRIDES
    rng = np.random.default_rng(B * 10 + ncls)
    hw = [(40, 64), (20, 32), (10, 16)]
    A = sum(h * w for h, w in hw)
    counts = [[0], [700, 0], [1500, 0, 300], [2000, 0, 1, 3360]][B - 1]
    ro, cl = _maps(B, hw, ncls, counts, rng)
    pred = ops.head_decode(ro, cl, hw, STRIDES, ncls).view(B, A, 5 + ncls)
    conf, thr = 0.05, 0.6
    refs = []
    for b in range(B):
        p = pred[b].cpu()
        det, _ = candidates(p, ncls, conf)
        s = (det[:, 4] * det[:, 5]).numpy()
        refs.append(reference(p, ncls, conf, thr, stable=len(np.unique(s)) < len(s)))
    for path in ("decoded", "fused"):
        for agn in (False, True):
            ws = ops.PostWorkspace(A, dev, B)
            if path == "decoded":
                post_ops.postprocess_device_ex(pred.contiguous(), ncls, conf, thr, ws, class_agnostic=agn)
            else:
                post_ops.det_candidates(ro, cl, hw, STRIDES, ncls, conf, ws)
                post_ops.postprocess_nms(thr, ws, class_agnostic=agn)
            cnt = ws.count.cpu().tolist()
            dets, anc = ws.dets.view(B, A, 7).cpu(), ws.anchors.view(B, A).cpu()
            for b in range(B):
                ref = refs[b] if not agn else reference(pred[b].cpu(), ncls, conf, thr, agnostic=True, stable=True)
                same((dets[b, :cnt[b]], anc[b, :cnt[b]]), ref, f"B={B} image {b} {path} {'agnostic' if agn else 'class-aware'}")
            assert cnt[min(1, B - 1)] == 0 and (B == 1 or min(cnt[:1] + cnt[2:]) > 0)


# ----------------------------------------------------------------------------------------------- decode
def test_head_decode_per_element_vs_float64():
    """uc_head_decode against float64: cx, cy bit-exact ((reg + grid) * stride, two roundings); w, h within expf's 2 ulp (the
    stride is a power of two); the sigmoids 1 / (1 + expf(-x)) within 6 ulp (expf's 2 ulp scaled by e / (1 + e) <= 1, plus the
    rounded add and divide: relative 3 * 2^-23 < 6 ulp).  Logits beyond the float range of exp: exp(x) > FLT_MAX for x > 88.72
    gives w = inf as torch.exp does; for x < -87.3 exp(x) is below FLT_MIN, and expf may return 0 where torch returns a
    denormal, so every bound has an absolute floor of 2^-126 (times the stride for w, h)."""
    from unicorn_b200.engine import STRIDES
    rng = np.random.default_rng(4)
    hw = [(24, 40), (12, 20), (6, 10)]
    ncls = 8
    ro, cl, ref_ro, ref_cl = [], [], [], []
    for h, w in hw:
        r = rng.normal(0, 3, (1, h, w, 5)).astype(f32)
        c = rng.normal(0, 6, (1, h, w, ncls)).astype(f32)
        flat = c.reshape(-1)
        flat[:200] = rng.uniform(-104, 104, 200)  # beyond the range of expf, both signs
        r.reshape(-1, 5)[:40, 2:] = rng.uniform(-100, 95, (40, 3))
        ro.append(torch.from_numpy(r).to(dev))
        cl.append(torch.from_numpy(c).to(dev))
    out = ops.head_decode(ro, cl, hw, STRIDES, ncls)[0].cpu().double()
    rows = []
    for (h, w), s, r, c in zip(hw, STRIDES, ro, cl):
        r, c = r[0].cpu().reshape(h * w, 5), c[0].cpu().reshape(h * w, ncls)
        yy, xx = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
        grid = torch.stack([xx, yy], -1).reshape(-1, 2).float()
        xy = (r[:, :2] + grid) * float(s)  # float32: the kernel's two roundings
        wh = torch.exp(r[:, 2:4].double()) * s
        sig = 1 / (1 + torch.exp(-torch.cat([r[:, 4:5], c], 1).double()))
        rows.append((xy, wh, sig, torch.full((h * w, 1), float(s), dtype=torch.float64)))
    xy = torch.cat([t[0] for t in rows])
    wh = torch.cat([t[1] for t in rows])
    sig = torch.cat([t[2] for t in rows])
    stride = torch.cat([t[3] for t in rows])
    assert torch.equal(out[:, :2].float(), xy)
    print(f"exact: {xy.numel()} cx, cy")

    def ulp(x):
        x32 = x.abs().float().clamp(min=2.0 ** -126)
        return (torch.nextafter(x32, torch.tensor(float("inf"))) - x32).double()

    def check(got, ref, n_ulp, floor, name):
        fin = ref <= float(np.finfo(f32).max)
        assert torch.equal(torch.isinf(got), ~fin), f"{name}: overflow differs"
        g, r, fl = got[fin], ref[fin], floor.expand_as(ref)[fin]
        err = (g - r).abs()
        ratio = (err / (n_ulp * ulp(r) + fl)).max().item()
        print(f"err/bound {ratio:.3f}  {name} ({int((~fin).sum())} overflow to inf, {int((r < fl).sum())} below the floor)")
        assert ratio <= 1.0, f"{name}: err/bound {ratio:.3g}"

    check(out[:, 2:4], wh, 2, stride * 2.0 ** -126, "w, h = expf(reg) * stride")
    check(out[:, 4:], sig, 6, torch.tensor(2.0 ** -126, dtype=torch.float64), "sigmoids of obj and classes")
    assert int((sig < 2.0 ** -126).sum()) > 10 and int((wh < 2.0 ** -126).sum()) > 0 and int((wh > float(np.finfo(f32).max)).sum()) > 0


# ----------------------------------------------------------------------------------------------- box IoU
def _iou_boxes(n, rng):
    q = 2.0 ** -11
    return random_boxes(n, rng, span=600.0) + np.float32(q) * rng.integers(0, 2, (n, 4)).astype(f32)


def test_box_iou_matches_torchvision_bit_for_bit():
    """plus_one = 0 against torchvision.ops.box_iou on CUDA and its float32 emulation; plus_one = 1 against the emulation of the
    same order, and within a derived bound of float64 bbox_overlaps (ByteTrack)."""
    rng = np.random.default_rng(8)
    a, b = _iou_boxes(300, rng), _iou_boxes(257, rng)
    ta, tb = torch.from_numpy(a).to(dev), torch.from_numpy(b).to(dev)
    got = ops.box_iou(ta, tb).cpu()
    tv = torchvision.ops.box_iou(ta, tb).cpu()
    emu = torch.from_numpy(orc.box_iou_f32(a, b))
    assert torch.equal(emu.view(torch.int32), tv.view(torch.int32))
    assert (tv > 0).sum() > 1000
    assert torch.equal(got.view(torch.int32), tv.view(torch.int32)), f"{int((got != tv).sum())} of {got.numel()} IoUs differ"
    print(f"exact: {got.numel()} box_iou values ({int((tv > 0).sum())} nonzero)")
    # strided rows (the tracker passes [N, 5] boxes with scores)
    a5 = torch.cat([ta, torch.rand(300, 1, device=dev)], 1)
    assert torch.equal(ops.box_iou(a5, tb).cpu(), got)

    got1 = ops.box_iou(ta, tb, plus_one=True).cpu().double()
    emu1 = torch.from_numpy(orc.box_iou_f32(a, b, plus_one=True)).double()
    assert torch.equal(got1, emu1)
    # float64 bbox_overlaps and a first-order bound of the float32 chain: every rounded step adds u = 2^-24 of its magnitude
    A, Bx = a.astype(np.float64), b.astype(np.float64)
    u = 2.0 ** -24
    wa, ha = A[:, 2] - A[:, 0] + 1, A[:, 3] - A[:, 1] + 1
    wb, hb = Bx[:, 2] - Bx[:, 0] + 1, Bx[:, 3] - Bx[:, 1] + 1
    d = [np.minimum(A[:, None, k + 2], Bx[None, :, k + 2]) - np.maximum(A[:, None, k], Bx[None, :, k]) for k in (0, 1)]
    iw, ih = d[0] + 1, d[1] + 1
    inter = np.where((iw > 0) & (ih > 0), iw * ih, 0.0)
    area = (wa * ha)[:, None] + (wb * hb)[None, :]
    union = area - inter
    ref = inter / union
    e_w = lambda dd, w: u * (np.abs(dd) + np.abs(w))  # noqa: E731  rn(rn(x2 - x1) + 1)
    e_area = lambda w, h, dw, dh: np.abs(h) * e_w(dw, w) + np.abs(w) * e_w(dh, h) + u * np.abs(w * h)  # noqa: E731
    e_a = e_area(wa, ha, wa - 1, ha - 1)[:, None] + e_area(wb, hb, wb - 1, hb - 1)[None, :]
    e_i = np.where(inter > 0, np.abs(ih) * e_w(d[0], iw) + np.abs(iw) * e_w(d[1], ih) + u * inter, 0.0)
    e_u = e_a + u * area + e_i + u * union
    bound = 1.01 * ((e_i + ref * e_u) / union + u * ref) + 1e-30
    err = np.abs(got1.numpy() - ref)
    ratio = (err / bound).max()
    print(f"err/bound {ratio:.3f}  box_iou plus_one=1 vs float64 bbox_overlaps (max err {err.max():.3g})")
    assert ratio <= 1.0

"""The COCO instance segmenter (unicorn_inst_convnext_tiny) on the H100: the 6-tuple, rows and masks against the reference golden
(tests/golden/inst_tiny_320.npz), the fused encode (uc_inst_encode_batched) string for string against uc_mots_encode of the
full-resolution masks and pixel for pixel against a torch restatement, and UnicornInstanceSegmenter's chunks, buffer growth and
batching.  The golden frame at conf 0.04 leaves 59 NMS rows; the driver tests run 320x320 inputs at conf 0.04 (a few dozen rows per
image)."""
import math
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
INST = "unicorn_inst_convnext_tiny"


@pytest.fixture(scope="module")
def golden():
    from test_inst import load_inst_golden
    return load_inst_golden()


@pytest.fixture(scope="module")
def model():
    from unicorn_b200.compat.model import UnicornB200Model
    from unicorn_b200.weights import make_state_dict
    return UnicornB200Model(make_state_dict(INST, 0), INST).eval()


def _frames(g, n=2):
    from unicorn_b200.synthetic import make_video
    frames, _ = make_video(n, 320, 320, seed=int(g["seed_video"]), n_obj=int(g["n_obj"]))
    return frames


def _run(e, img, conf, nms):
    """Backbone, head with controllers, fused candidates + class-aware NMS and the mask branch of B images."""
    from unicorn_b200 import ops, post_ops
    from unicorn_b200.engine import STRIDES
    from unicorn_b200.frames import anchor_count
    B, _, H, W = img.shape
    ws = ops.PostWorkspace(anchor_count(H, W), img.device, B)
    e.begin_frame()
    fpn, _ = e.backbone(img, tag="insttest")
    e.head(fpn, None, "mot", decode=False, with_masks=True)
    ro, cl, hw = e.head_maps
    post_ops.det_candidates(ro, cl, hw, STRIDES, 80, conf, ws)
    post_ops.postprocess_nms(nms, ws)
    mf, um = e.mask_branch(fpn)
    return ws, mf, um, list(e.dyn_levels)


def _fused(ws, mf, um, dyn, n_max, sizes, ratios, thr, capacity=1 << 16):
    """The first n_max rows' strings of every image through dynamic_masks_rows + uc_inst_encode_batched."""
    from unicorn_b200 import post_ops
    from unicorn_b200.mots import MaskEncoder
    B, h, w, _ = mf.shape
    maps = torch.empty(B, n_max, h * 4, w * 4, device="cuda")
    window = ws.count.clamp(max=n_max).to(torch.int32)
    post_ops.dynamic_masks_rows(mf, um, dyn, [(t.shape[1], t.shape[2]) for t in dyn], ws.anchors.view(B, -1), window,
                                torch.arange(B, dtype=torch.int32, device="cuda"), n_max, 4, maps, torch.empty(B * n_max * h * w, device="cuda"))
    enc = MaskEncoder(B * n_max, "cuda", capacity)
    enc.reserve(max(s[0] for s in sizes), max(s[1] for s in sizes))
    run = lambda: post_ops.inst_encode(maps, ws.count, 0, 2, thr, ratios, [s[0] for s in sizes], [s[1] for s in sizes], enc.ws,  # noqa: E731
                                       enc.d_emit, enc.d_chars, enc.d_offsets)
    enc.enqueue(B * n_max, run)
    flat = enc.strings(B * n_max, run)
    counts = ws.count.tolist()
    return [flat[b * n_max:b * n_max + min(n_max, counts[b])] for b in range(B)], maps


def _iou(a, b):
    return (a & b).sum() / max((a | b).sum(), 1)


def test_inst_head_rows_and_masks_vs_reference_golden(model, golden):
    import unicorn_oracle as orc
    from test_det_gpu import check_dets_80
    from test_whole_gpu import check_head
    from unicorn_b200.compat.model import postprocess_inst
    from unicorn_b200.results import rle_decode
    g = golden
    f = int(g["frame"])
    img = _frames(g)[f:f + 1].cuda()
    out, locs, dyn, lvls, mf, um = model(img)
    check_head(out, g["head"])
    assert torch.equal(locs.cpu(), torch.from_numpy(g["locations"])) and torch.equal(lvls.cpu(), torch.from_numpy(g["fpn_levels"]))
    rel = lambda a, b: ((a.float().cpu() - b).abs().max() / (b.abs().max() + 1e-12)).item()  # noqa: E731
    assert dyn.shape == (1, 2100, 169) and rel(dyn[0, ::16], torch.from_numpy(g["dyn_sub"])) < 8e-2
    assert mf.shape == (1, 8, 40, 40) and rel(mf, torch.from_numpy(g["mask_feats"])) < 8e-2
    assert um.shape == (1, 144, 40, 40) and rel(um[0, :, ::4, ::4], torch.from_numpy(g["up_masks_sub"])) < 8e-2
    conf, nms, thr = float(g["conf"]), float(g["nms"]), float(g["thr"])
    dets, masks = postprocess_inst(out.clone(), locs, dyn, lvls, mf, model.head.mask_head, 80, conf, nms, d_rate=2, up_masks=um)
    dets, masks = dets[0].cpu(), masks[0]
    ref = torch.from_numpy(g["dets"])
    check_dets_80(dets, ref, g["head"], orc)
    assert masks.shape == (dets.shape[0], 1, 320, 320)
    # the fused path on the same frame (original size = input size, r = 1: the resize is the identity)
    ws, mf2, um2, dyn2 = _run(model.engine, img, conf, nms)
    rows = ws.dets.view(1, -1, 7)[0, :int(ws.count[0])].cpu()
    assert rows.shape == dets.shape and torch.equal(rows[:, 6], dets[:, 6]) and (rows - dets).abs().max() < 1e-4
    rles, _ = _fused(ws, mf2, um2, dyn2, 128, [(320, 320)], [1.0], thr)
    # a row's mask depends on its anchor (controller outputs, location): compare the rows whose anchor the reference kept too (the
    # anchor of a reference row is the one whose decoded corners it holds)
    href = torch.from_numpy(g["head"])[0]
    corners = torch.stack([href[:, 0] - href[:, 2] / 2, href[:, 1] - href[:, 3] / 2, href[:, 0] + href[:, 2] / 2, href[:, 1] + href[:, 3] / 2], 1)
    ref_row = {int((corners - ref[j, :4]).abs().sum(1).argmin()): j for j in range(ref.shape[0])}
    anchors = ws.anchors.view(1, -1)[0, :dets.shape[0]].tolist()
    # and whose reference mask is well conditioned: under 5 % of its pixels within 0.05 of the threshold.  The seeded weights give
    # some rows flat masks, where the engine's bf16 controller outputs (within 8e-2 of the reference) move large areas across it.
    matched, ious = 0, []
    for i, a in enumerate(anchors):
        if a not in ref_row:
            continue
        j = ref_row[a]
        want = rle_decode(g["rles"][j], 320, 320)
        got = rle_decode(rles[0][i], 320, 320)
        assert np.array_equal(got, (masks[i, 0] > thr).cpu().numpy())  # the fused encode is postprocess_inst's mask, thresholded
        ious.append((round(float(_iou(got, want)), 4), round(float(g["near_thr"][j]), 4)))
        if g["near_thr"][j] < 0.05:
            assert _iou(got, want) >= 0.95, (i, a, ious[-1])
            matched += 1
    print("mask IoU, near-threshold fraction of the reference:", ious)
    assert matched >= 0.5 * dets.shape[0], (matched, dets.shape[0])


SIZES = [[(320, 320), (337, 200)], [(480, 640), (320, 320)], [(337, 200), (480, 640)]]


@pytest.mark.parametrize("thr", [0.3, 0.5])
@pytest.mark.parametrize("sizes", SIZES)
def test_fused_encode_equals_mots_encode_of_full_resolution_masks(model, golden, thr, sizes):
    """Two images of a batch at (320, 320) (r = 1), (480, 640) (r = 0.5) and (337, 200), whose resize is one row short (floor(320 *
    (1 / (320 / 337))) = 336): every string equals uc_mots_encode of that one instance of dynamic_masks(d_rate=2), padded with
    background to the whole frame, and the decoded masks equal a torch F.interpolate restatement except within 1e-5 of thr."""
    from unicorn_b200 import ops
    from unicorn_b200.mots import MaskEncoder
    from unicorn_b200.results import rle_decode, rle_encode
    img = _frames(golden)[0:2].cuda()
    ws, mf, um, dyn = _run(model.engine, img, float(golden["conf"]), float(golden["nms"]))
    ratios = [min(320 / float(h), 320 / float(w)) for h, w in sizes]
    n_max = 64
    fused, _ = _fused(ws, mf, um, dyn, n_max, sizes, ratios, thr)
    full = ops.dynamic_masks(mf, um, dyn, [(t.shape[1], t.shape[2]) for t in dyn], ws, n_max, up_rate=4, d_rate=2)
    enc = MaskEncoder(1, "cuda")
    checked = 0
    for b, ((H, W), r) in enumerate(zip(sizes, ratios)):
        hm, wm = min(H, math.floor(320 * (1.0 / r))), min(W, math.floor(320 * (1.0 / r)))
        assert (hm < H) == ((H, W) == (337, 200))
        for i, s in enumerate(fused[b]):
            ref = enc(full[b], [i], [True], thr, r, H, W)[0]
            if (hm, wm) == (H, W):
                assert s == ref, (b, i)
            pad = np.zeros((H, W), dtype=bool)
            pad[:hm, :wm] = rle_decode(ref, hm, wm)
            assert s == rle_encode(pad), (b, i)
            v = F.interpolate(full[b, i][None, None], scale_factor=1 / r, mode="bilinear", align_corners=False)[0, 0, :H, :W].cpu()
            soft = torch.zeros(H, W)
            soft[:v.shape[0], :v.shape[1]] = v
            diff = torch.from_numpy(rle_decode(s, H, W)) != (soft > thr)
            assert not diff[(soft - thr).abs() >= 1e-5].any(), (b, i)
            checked += 1
        assert len(fused[b]) == min(n_max, int(ws.count[b]))
    assert checked >= 40


def _images(seed=5):
    from unicorn_b200.synthetic import make_video
    out = []
    for k, (h, w) in enumerate([(480, 640), (337, 200), (320, 320)]):
        f, _ = make_video(1, h, w, seed=seed + k, n_obj=4)
        out.append(f[0].permute(1, 2, 0).round().clamp(0, 255).to(torch.uint8).numpy())
    return out


def _same(a, b):
    assert len(a) == len(b)
    for (ra, sa, la), (rb, sb, lb) in zip(a, b):
        assert sa == sb and torch.equal(ra, rb) and la == lb


@pytest.fixture(scope="module")
def seg_engine(model):
    return model.engine


def test_segmenter_chunks_capacity_and_partial_batches(seg_engine):
    from unicorn_b200.det import UnicornInstanceSegmenter
    from unicorn_b200.results import rle_decode
    e, ims = seg_engine, _images()
    kw = dict(input_size=(320, 320), conf=0.04, nms=0.65)
    one = UnicornInstanceSegmenter(e, max_batch=1, chunk=256, **kw)
    alone = [one.detect([im])[0] for im in ims]
    for (rows, r, rles), im in zip(alone, ims):
        h, w = im.shape[:2]
        assert 16 < rows.shape[0] <= 256 and len(rles) == rows.shape[0] and r == min(320 / h, 320 / w)
        assert all(rle_decode(s, h, w).shape == (h, w) for s in rles)
        assert sum(rle_decode(s, h, w).any() for s in rles) > rows.shape[0] // 2
    # chunks of 16 rows and a 1-byte initial chars buffer give the same rows and strings
    _same([UnicornInstanceSegmenter(e, max_batch=1, chunk=16, **kw).detect([im])[0] for im in ims], alone)
    _same([UnicornInstanceSegmenter(e, max_batch=1, chunk=256, capacity=1, **kw).detect([im])[0] for im in ims], alone)
    # a partial batch of mixed sizes, in graph and eager mode, with chunks: each image as in its own one-image run
    for use_graph in (True, False):
        seg = UnicornInstanceSegmenter(e, max_batch=3, chunk=16, use_graph=use_graph, **kw)
        _same(seg.detect(ims[:2]), alone[:2])
        _same(seg.detect(ims), alone)
        _same(seg.detect(ims[1:2]), alone[1:2])
    # two steps in flight on two streams
    seg = UnicornInstanceSegmenter(e, max_batch=2, chunk=16, depth=2, **kw)
    seg.submit(ims[:2])
    seg.submit(ims[2:])
    _same(seg.collect(), alone[:2])
    _same(seg.collect(), alone[2:])


def test_segmenter_rejects_non_mask_configs(seg_engine):
    from unicorn_b200.det import UnicornInstanceSegmenter
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.weights import make_state_dict
    with pytest.raises(ValueError, match="instance-segmentation"):
        UnicornInstanceSegmenter(UnicornEngine(make_state_dict("unicorn_det_convnext_tiny", 0), "unicorn_det_convnext_tiny"))
    with pytest.raises(ValueError, match="d_rate"):
        UnicornInstanceSegmenter(seg_engine, d_rate=4)

"""NV12 frames on the H100: uc_letterbox_nv12 against the reference path for an NV12 frame (cv2.cvtColor(COLOR_YUV2RGB_NV12), then
the SOT preprocessor) on pitched rows, separate planes and a non-default pad, and every driver that takes raw frames giving, for NV12
frames, exactly what it gives for the same frames converted to RGB with cv2 (CUDA graphs on), with RGB and NV12 frames mixed in one
batched step and malformed 2-D frames rejected without a trace."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_nv12 import SOURCES, TARGETS, nv12_frame  # noqa: E402

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
TINY = (320, 320)


def rgb_of(nv12):
    return cv2.cvtColor(nv12, cv2.COLOR_YUV2RGB_NV12)


def recipe(nv12, size):
    """The reference path: cv2's RGB frame through the SOT preprocessor."""
    from unicorn_b200.sot import preprocess
    return preprocess(rgb_of(nv12), size, out=torch.empty(1, *size, 3, dtype=torch.uint8))


def nv12_of(rgb):
    """An NV12 frame of an RGB image (h a multiple of 4, w even), through cv2's I420 encoder."""
    h, w = rgb.shape[:2]
    i420 = cv2.cvtColor(np.ascontiguousarray(rgb), cv2.COLOR_RGB2YUV_I420)
    u, v = i420[h:h + h // 4].reshape(h // 2, w // 2), i420[h + h // 4:].reshape(h // 2, w // 2)
    nv = np.empty((h * 3 // 2, w), dtype=np.uint8)
    nv[:h] = i420[:h]
    nv[h:] = np.stack([u, v], -1).reshape(h // 2, w)
    return nv


def video_nv12(n, h, w, seed, n_obj=2):
    """n NV12 frames of a synthetic video (structured content), their cv2 RGB frames and the objects' boxes (xyxy, original pixels)."""
    from unicorn_b200.synthetic import make_video
    frames, boxes = make_video(n, h, w, seed=seed, n_obj=n_obj)
    nv = [nv12_of(f.permute(1, 2, 0).flip(-1).round().clamp(0, 255).to(torch.uint8).numpy()) for f in frames]
    return nv, [rgb_of(f) for f in nv], boxes


def xywh(b):
    return [float(b[0]), float(b[1]), float(b[2] - b[0]), float(b[3] - b[1])]


_ENGINES = {}


def engine(name):
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.weights import make_state_dict
    if name not in _ENGINES:
        _ENGINES.clear()  # one engine alive at a time
        _ENGINES[name] = UnicornEngine(make_state_dict(name, 0), name)
    return _ENGINES[name]


# ---------------------------------------------------------------------------------------------------------------- kernel
@pytest.mark.parametrize("size", TARGETS)
@pytest.mark.parametrize("hw", SOURCES)
def test_kernel_equals_cv2_recipe(hw, size):
    from unicorn_b200 import shared_ops
    nv12 = nv12_frame(*hw, seed=hw[0] + 3 * hw[1])
    ref, r = recipe(nv12, size)
    out, r2 = shared_ops.letterbox_nv12(torch.from_numpy(nv12).cuda(), size)
    assert r2 == r
    assert torch.equal(out.cpu(), ref)


@pytest.mark.parametrize("hw,size", [((1080, 1920), (800, 1280)), ((362, 498), (320, 320)), ((2, 2), (320, 320))])
def test_kernel_pitched_rows_and_pad_touch_only_the_slot(hw, size):
    """src a view of a wider buffer (row pitch > w, offset columns), pad 7, out the middle slot of three: equal to the recipe with
    pad 7, and the neighbouring slots keep their bytes."""
    import nv12_oracle
    from unicorn_b200 import shared_ops
    h, w = hw
    nv12 = nv12_frame(h, w, seed=9)
    wide = torch.randint(0, 256, (h * 3 // 2, w + 72), dtype=torch.uint8, device="cuda")
    wide[:, 40:40 + w] = torch.from_numpy(nv12).cuda()
    big = torch.randint(0, 256, (3, *size, 3), dtype=torch.uint8, device="cuda")
    before = big.clone()
    out, r = shared_ops.letterbox_nv12(wide[:, 40:40 + w], size, pad=7, out=big[1:2])
    want, r2 = nv12_oracle.letterbox_nv12(nv12, size, pad=7)
    assert r == r2 == recipe(nv12, size)[1]
    rh, rw = int(h * r), int(w * r)
    assert torch.equal(out[0, :rh, :rw].cpu(), recipe(nv12, size)[0][0, :rh, :rw])
    assert torch.equal(big[1].cpu(), torch.from_numpy(want))
    assert torch.equal(big[0], before[0]) and torch.equal(big[2], before[2])


def test_kernel_separate_planes_with_padding_rows():
    """A decoder surface: Y plane, 8 padding rows, then the UV plane, row pitch 2048 for a 1920-wide frame, through the C ABI."""
    from unicorn_b200 import _lib
    h, w, ld, gap = 1080, 1920, 2048, 8
    nv12 = nv12_frame(h, w, seed=21)
    surf = torch.randint(0, 256, (h + gap + h // 2, ld), dtype=torch.uint8, device="cuda")
    surf[:h, :w] = torch.from_numpy(nv12[:h]).cuda()
    surf[h + gap:, :w] = torch.from_numpy(nv12[h:]).cuda()
    H, W = 800, 1280
    ref, r = recipe(nv12, (H, W))
    out = torch.empty(1, H, W, 3, dtype=torch.uint8, device="cuda")
    rc = _lib.lib().uc_letterbox_nv12(ctypes.c_void_p(surf.data_ptr()), ctypes.c_void_p(surf[h + gap].data_ptr()), ld, h, w,
                                      ctypes.c_void_p(out.data_ptr()), H, W, int(h * r), int(w * r), 114, _lib.stream_ptr())
    _lib.check(rc, "uc_letterbox_nv12")
    assert torch.equal(out.cpu(), ref)


# ---------------------------------------------------------------------------------------------------------------- drivers
@pytest.mark.parametrize("device_preproc", [False, True])
def test_sot_batch(device_preproc):
    """Two sequences: NV12 host arrays, NV12 CUDA tensors and RGB / NV12 mixed per step give the boxes of the cv2 RGB frames."""
    from unicorn_b200.sot import UnicornSOTBatch
    e = engine("unicorn_track_tiny")
    vids = [video_nv12(5, 240, 400, seed=1), video_nv12(5, 320, 256, seed=2)]

    def run(pick):
        b = UnicornSOTBatch(e, TINY, 2, device_preproc=device_preproc)
        for i, (nv, rgb, boxes) in enumerate(vids):
            b.initialize(i, pick(i, 0, nv[0], rgb[0]), {"init_bbox": xywh(boxes[0, 0])})
        out = []
        for t in range(1, 5):
            res = b.track([pick(i, t, nv[t], rgb[t]) for i, (nv, rgb, _) in enumerate(vids)])
            counts = b.slot.host_count.tolist()
            out.append((res, counts, [b.slot.host_dets[i, :min(c, b.max_inst)].tolist() for i, c in enumerate(counts)]))
        return out
    want = run(lambda i, t, nv, rgb: rgb)
    assert all(c > 0 for _, counts, _ in want for c in counts)  # every step of both sequences has detections to compare
    assert run(lambda i, t, nv, rgb: nv) == want
    assert run(lambda i, t, nv, rgb: torch.from_numpy(nv).cuda()) == want
    assert run(lambda i, t, nv, rgb: nv if (i + t) % 2 else rgb) == want


def test_vos_track_and_batch():
    """UnicornVOSTrack and UnicornVOSBatch (graphs on): label maps, soft masks, detection rows and states of NV12 frames equal those of
    the cv2 RGB frames; the batch mixes RGB and NV12 frames in a step."""
    from unicorn_b200.vos import UnicornVOSBatch, UnicornVOSTrack
    e = engine("unicorn_track_tiny_mask")
    vids = [video_nv12(4, 240, 400, seed=3), video_nv12(4, 480, 640, seed=4)]
    info = lambda boxes: {"init_object_ids": [1, 2], "init_bbox": {1: xywh(boxes[0, 0]), 2: xywh(boxes[0, 1])}}  # noqa: E731

    def track(pick):
        trk = UnicornVOSTrack(e, TINY, use_graph=True)
        nv, rgb, boxes = vids[0]
        trk.initialize(pick(0, nv[0], rgb[0]), info(boxes))
        out = []
        for t in range(1, 4):
            seg = trk.track(pick(t, nv[t], rgb[t]))["segmentation"]
            out.append((seg, trk._soft[:2].cpu(), trk._workers[0].rows_host[:2].clone(), dict(trk.state_pre_dict)))
        return out

    def batch(pick):
        b = UnicornVOSBatch(e, TINY, 2, 4, 2)
        for i, (nv, rgb, boxes) in enumerate(vids):
            b.initialize(i, pick(i, nv[0], rgb[0]), info(boxes))
        out = []
        for t in range(1, 4):
            segs = b.track([pick(i + t, nv[t], rgb[t]) for i, (nv, rgb, _) in enumerate(vids)])
            out.append(([s["segmentation"] for s in segs], [sq.soft[:2].cpu() for sq in b.seqs], b.host_rows.clone(),
                        [dict(d) for d in b.state_pre_dicts]))
        return out

    def same(a, b):
        for x, y in zip(a, b):
            for u, v in zip(x, y):
                if isinstance(u, list):
                    assert all(np.array_equal(p, q) if isinstance(p, np.ndarray) else (torch.equal(p, q) if torch.is_tensor(p) else p == q)
                               for p, q in zip(u, v))
                elif isinstance(u, np.ndarray):
                    assert np.array_equal(u, v)
                elif torch.is_tensor(u):
                    assert torch.equal(u, v)
                else:
                    assert u == v
    want = track(lambda t, nv, rgb: rgb)
    same(track(lambda t, nv, rgb: nv), want)
    assert want[-1][0].max() > 0
    want = batch(lambda k, nv, rgb: rgb)
    same(batch(lambda k, nv, rgb: nv), want)
    same(batch(lambda k, nv, rgb: nv if k % 2 else rgb), want)


def test_unified_batch():
    from test_unified_mask_gpu import qd_tracker
    from unicorn_b200.unified import UnicornUnifiedBatch
    e = engine("unicorn_track_tiny")
    vids = [video_nv12(4, 240, 400, seed=5), video_nv12(4, 320, 256, seed=6)]

    def run(pick):
        b = UnicornUnifiedBatch(e, TINY, 2, 4, mot="qd", mot_conf=0.01, score_thr=0.02)
        for i in range(2):
            b.start(i, qd_tracker())
        out = []
        for t in range(4):
            new = {i: {1: xywh(boxes[0, 0])} for i, (_, _, boxes) in enumerate(vids)} if t == 0 else None
            res = b.track([pick(i + t, nv[t], rgb[t]) for i, (nv, rgb, _) in enumerate(vids)], new)
            out.append([(r["targets"], [m.clone() for m in r["mot"]]) for r in res])
        return out

    def same(a, b):
        for x, y in zip(a, b):
            for (ta, ma), (tb, mb) in zip(x, y):
                assert ta == tb and all(torch.equal(p, q) for p, q in zip(ma, mb))
    want = run(lambda k, nv, rgb: rgb)
    same(run(lambda k, nv, rgb: nv), want)
    same(run(lambda k, nv, rgb: nv if k % 2 else rgb), want)


def test_unified_mask_batch_full_hd_and_vga():
    """A 1080x1920 and a 480x640 video in one batch: label maps, MOTS tuples and states of NV12 frames equal the cv2 RGB frames'."""
    from test_unified_mask_gpu import MOTS_KW, qd_tracker
    from unicorn_b200.unified import UnicornUnifiedMaskBatch
    e = engine("unicorn_track_tiny_mask")
    vids = [video_nv12(3, 1080, 1920, seed=7), video_nv12(3, 480, 640, seed=8)]

    def run(pick):
        b = UnicornUnifiedMaskBatch(e, TINY, 2, 4, 2, **MOTS_KW)
        for i, (nv, _, _) in enumerate(vids):
            b.start(i, (nv[0].shape[0] * 2 // 3, nv[0].shape[1]), qd_tracker())
        out = []
        for t in range(3):
            infos = [{"init_object_ids": [1], "init_bbox": {1: xywh(boxes[0, 0])}} if t == 0 else None for _, _, boxes in vids]
            res = b.track([pick(i + t, nv[t], rgb[t]) for i, (nv, rgb, _) in enumerate(vids)], infos)
            out.append(([r["segmentation"] for r in res], [r["mots"] for r in res], [dict(d) for d in b.state_pre_dicts]))
        return out

    def same(a, b):
        for (sa, ma, da), (sb, mb, db) in zip(a, b):
            assert all(np.array_equal(p, q) for p, q in zip(sa, sb)) and ma == mb and da == db
    want = run(lambda k, nv, rgb: rgb)
    same(run(lambda k, nv, rgb: nv), want)
    same(run(lambda k, nv, rgb: torch.from_numpy(nv).cuda() if k % 2 else rgb), want)
    assert want[-1][0][0].max() > 0


def _images():
    return [video_nv12(1, h, w, seed=30 + k, n_obj=4)[:2] for k, (h, w) in enumerate([(480, 640), (336, 200), (320, 320)])]


def _same_rows(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert x[1] == y[1] and torch.equal(x[0], y[0]) and x[2:] == y[2:]


@pytest.mark.parametrize("name,segmenter", [("unicorn_det_convnext_tiny", False), ("unicorn_inst_convnext_tiny", True)])
def test_detector_and_segmenter_mixed_sizes(name, segmenter):
    """A batch of three sizes: NV12 frames give the rows (and RLE strings) of their cv2 RGB frames with rgb=True, also mixed."""
    from unicorn_b200.det import UnicornDetector, UnicornInstanceSegmenter
    e = engine(name)
    ims = _images()
    nv, rgb = [v[0][0] for v in ims], [v[1][0] for v in ims]
    det = (UnicornInstanceSegmenter(e, TINY, max_batch=3, conf=0.04, chunk=16) if segmenter else
           UnicornDetector(e, TINY, max_batch=3, conf=0.04))
    want = det.detect(rgb, rgb=True)
    assert all(w[0].shape[0] > 0 for w in want)
    _same_rows(det.detect(nv), want)
    _same_rows(det.detect([nv[0], rgb[1], torch.from_numpy(nv[2]).cuda()], rgb=True), want)


def test_detector_in_flight_frames_dropped_after_submit():
    """depth = 2: CUDA NV12 and RGB frames the caller drops right after submit(), their memory then taken by new tensors filled on
    the default stream, still give the rows of frames the caller keeps."""
    from unicorn_b200.det import UnicornDetector
    e = engine("unicorn_det_convnext_tiny")
    ims = _images()
    nv, rgb = [v[0][0] for v in ims], [v[1][0] for v in ims]
    det = UnicornDetector(e, TINY, max_batch=3, conf=0.04, depth=2)
    want = det.detect(rgb, rgb=True)
    for _ in range(3):
        det.submit([torch.from_numpy(nv[0]).cuda(), torch.from_numpy(rgb[1]).cuda(), torch.from_numpy(nv[2]).cuda()], rgb=True)
        det.submit([torch.from_numpy(f).cuda() for f in rgb], rgb=True)
        junk = [torch.full((f.size,), 255, dtype=torch.uint8, device="cuda") for f in nv + rgb]  # takes the dropped blocks if free
        _same_rows(det.collect(), want)
        _same_rows(det.collect(), want)
        del junk


# ---------------------------------------------------------------------------------------------------------------- rejection
BAD = [np.zeros((5, 4), np.uint8), np.zeros((6, 3), np.uint8), np.zeros((6, 4), np.float32)]


def test_malformed_frames_are_rejected_and_drivers_stay_usable():
    from test_unified_mask_gpu import MOTS_KW
    from unicorn_b200.det import UnicornDetector
    from unicorn_b200.sot import UnicornSOTBatch
    from unicorn_b200.unified import UnicornUnifiedMaskBatch
    nv, rgb, boxes = video_nv12(3, 240, 400, seed=11)
    e = engine("unicorn_track_tiny")
    sot = UnicornSOTBatch(e, TINY, 2)
    for i in range(2):
        sot.initialize(i, nv[0], {"init_bbox": xywh(boxes[0, 0])})
    for bad in BAD:
        with pytest.raises(ValueError, match="NV12"):
            sot.initialize(0, bad, {"init_bbox": [0, 0, 4, 4]})
        with pytest.raises(ValueError, match="NV12"):
            sot.track([nv[1], bad])
    assert sot.track([nv[1], rgb[1]])[0] == sot.track([rgb[1], nv[1]])[1]

    e = engine("unicorn_track_tiny_mask")
    b = UnicornUnifiedMaskBatch(e, TINY, 2, 4, 2, **MOTS_KW)
    b.start(0, (240, 400))
    b.start(1, (240, 400))
    before = (b._ring.submitted, list(b.frame_ids), list(b._os))
    for bad in BAD:
        with pytest.raises(ValueError, match="NV12"):
            b.track([nv[0], bad], [{"init_object_ids": [1], "init_bbox": {1: xywh(boxes[0, 0])}}, None])
    with pytest.raises(ValueError, match="size"):
        b.track([nv[0], nv12_frame(480, 640, 1)])  # a valid NV12 frame of the wrong size
    assert (b._ring.submitted, list(b.frame_ids), list(b._os)) == before
    out = b.track([nv[0], rgb[0]], [{"init_object_ids": [1], "init_bbox": {1: xywh(boxes[0, 0])}}] * 2)
    assert np.array_equal(out[0]["segmentation"], out[1]["segmentation"])

    e = engine("unicorn_det_convnext_tiny")
    det = UnicornDetector(e, TINY, max_batch=2, conf=0.04)
    for bad in BAD:
        with pytest.raises(ValueError, match="NV12"):
            det.detect([nv[0], bad])
    assert det._ring.submitted == det._ring.collected == 0
    a, c = det.detect([nv[0], rgb[0]], rgb=True)
    assert torch.equal(a[0], c[0]) and a[1] == c[1]

"""The COCO detectors on the H100: heads against the reference goldens (tests/golden/det_*_320.npz), the fused candidate filter
bit for bit against head_decode + the filter of postprocess, class-agnostic NMS against a greedy reference, and UnicornDetector's
batching (partial batches, mixed image sizes, graph and eager)."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

MODELS = [("tiny", "unicorn_det_convnext_tiny"), ("r50", "unicorn_det_r50"), ("large", "unicorn_det_convnext_large")]


@pytest.mark.parametrize("tag,name", MODELS)
def test_det_head_and_detections_vs_reference_golden(tag, name):
    import unicorn_oracle as orc
    from test_whole_gpu import check_head
    from unicorn_b200.compat.model import UnicornB200Model, postprocess
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.weights import make_state_dict
    g = np.load(os.path.join(ROOT, "tests", "golden", f"det_{tag}_320.npz"))
    frames, _ = make_video(2, 320, 320, seed=int(g["seed_video"]), n_obj=int(g["n_obj"]))
    img = frames[int(g["frame"]):int(g["frame"]) + 1].cuda()
    model = UnicornB200Model(make_state_dict(name, 0), name).eval()
    head = model(img)
    check_head(head, g["head"])
    e = model.engine  # model(imgs) is the engine's head output
    e.begin_frame()
    fpn, _ = e.backbone(img, tag="check")
    assert torch.equal(e.head(fpn, None, "mot"), head)
    dets = postprocess(head.clone(), 80, float(g["conf"]), float(g["nms"]))[0]
    check_dets_80(dets.cpu(), torch.from_numpy(g["dets"]), g["head"], orc)
    dets = postprocess(head.clone(), 80, float(g["conf_agnostic"]), float(g["nms_agnostic"]), class_agnostic=True)[0]
    ref = torch.from_numpy(g["dets_agnostic"])
    assert abs(dets.shape[0] - ref.shape[0]) <= max(5, 0.05 * ref.shape[0]), (dets.shape, ref.shape)


def check_dets_80(dets, ref, href, orc):
    """test_whole_gpu.check_dets for an 80-class head: counts within 5 %, and every engine row with score > 0.05 lies on a reference
    row (IoU > 0.7, score within 5e-2) of the same class, or of a class the reference itself scores within the probability tolerance
    (5e-2) of the engine's: with 80 classes the best two class probabilities of an anchor are often that close, and the argmax flips."""
    n = dets.shape[0]
    assert abs(n - ref.shape[0]) <= max(5, 0.05 * ref.shape[0]), (n, ref.shape[0])
    iou = orc.box_iou_np(dets[:, :4].numpy(), ref[:, :4].numpy())
    strong = np.nonzero((dets[:, 4] * dets[:, 5]).numpy() > 0.05)[0]
    assert (iou.max(1)[strong] > 0.7).all(), iou.max(1)[strong]
    href = torch.as_tensor(href)[0]
    corners = torch.stack([href[:, 0] - href[:, 2] / 2, href[:, 1] - href[:, 3] / 2, href[:, 0] + href[:, 2] / 2, href[:, 1] + href[:, 3] / 2], 1)
    for i in strong:
        j = int(iou[i].argmax())
        c_eng, c_ref = int(dets[i, 6]), int(ref[j, 6])
        if c_eng != c_ref:
            a = int((corners - ref[j, :4]).abs().sum(1).argmin())  # the reference row's anchor
            assert href[a, 5 + c_ref] - href[a, 5 + c_eng] < 5e-2, (i, c_eng, c_ref, href[a, 5 + c_ref].item(), href[a, 5 + c_eng].item())
    j = iou.argmax(1)
    sc, sr = (dets[:, 4] * dets[:, 5]).numpy(), (ref[:, 4] * ref[:, 5]).numpy()[j]
    assert np.abs(sc - sr)[iou.max(1) > 0.7].max() < 5e-2


def _maps(B, H, W, ncls, ld_cls, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    ro, cl, hw = [], [], []
    for s in (8, 16, 32):
        h, w = H // s, W // s
        r = torch.randn(B, h, w, 8, device="cuda", generator=g) * 0.5
        r[..., 4] = torch.randn(B, h, w, device="cuda", generator=g) * 2 - 2
        c = torch.randn(B, h, w, ld_cls, device="cuda", generator=g) * 3 - 4
        if ncls > 5:  # saturated logits: classes 3 and 5 both have sigmoid 1.0f, the first index must win though logit 5 is larger
            c[:, ::3, ::2, 3] = 18.0
            c[:, ::3, ::2, 5] = 30.0
        ro.append(r); cl.append(c); hw.append((h, w))
    return ro, cl, hw


def _slices(ws, B, A):
    """Per image: (count, det rows [A, 7], keys [a2], det_anchor [A]) views of the workspace."""
    a2 = 1
    while a2 < A:
        a2 <<= 1
    per = ws.nbytes // B
    out = []
    for b in range(B):
        s = ws.buf[b * per:(b + 1) * per]
        det0 = 256
        key0 = det0 + 2 * A * 28
        anc0 = key0 + a2 * 8
        out.append((s[:4].view(torch.int32)[0].item(), s[det0:det0 + A * 28].view(torch.float32).view(A, 7),
                    s[key0:key0 + a2 * 8].view(torch.int64), s[anc0:anc0 + A * 4].view(torch.int32)))
    return out


@pytest.mark.parametrize("B,ncls,ld_cls", [(1, 80, 80), (3, 80, 80), (1, 1, 8), (3, 8, 8), (2, 1, 8)])
def test_fused_candidates_bit_identical_to_decode_and_filter(B, ncls, ld_cls):
    from unicorn_b200 import ops, post_ops
    from unicorn_b200.engine import STRIDES
    H, W = 800, 1280
    ro, cl, hw = _maps(B, H, W, ncls, ld_cls, seed=B * 100 + ncls)
    A = sum(h * w for h, w in hw)
    ws1, ws2 = ops.PostWorkspace(A, "cuda", B), ops.PostWorkspace(A, "cuda", B)
    pred = ops.head_decode(ro, cl, hw, STRIDES, ncls)
    if B == 1:
        pred = pred.view(1, A, 5 + ncls)
    post_ops.postprocess_device_ex(pred, ncls, 0.01, 0.65, ws1)
    post_ops.det_candidates(ro, cl, hw, STRIDES, ncls, 0.01, ws2)
    post_ops.postprocess_nms(0.65, ws2)
    torch.cuda.synchronize()
    for (n1, d1, k1, a1), (n2, d2, k2, a2) in zip(_slices(ws1, B, A), _slices(ws2, B, A)):
        assert n1 == n2 and n1 > 0
        assert torch.equal(d1[:n1].view(torch.int32), d2[:n2].view(torch.int32))
        assert torch.equal(k1[:n1], k2[:n2]) and torch.equal(a1[:n1], a2[:n2])
    assert torch.equal(ws1.count, ws2.count)
    cnt = ws1.count.tolist()
    d1, d2 = ws1.dets.view(B, A, 7), ws2.dets.view(B, A, 7)
    x1, x2 = ws1.anchors.view(B, A), ws2.anchors.view(B, A)
    for b, n in enumerate(cnt):
        assert torch.equal(d1[b, :n].view(torch.int32), d2[b, :n].view(torch.int32)) and torch.equal(x1[b, :n], x2[b, :n])
    if ncls > 5:  # the saturated anchors are candidates with class 3
        d = d1[0, :cnt[0]]
        assert ((d[:, 5] == 1.0) & (d[:, 6] == 3.0)).any() and not ((d[:, 5] == 1.0) & (d[:, 6] == 5.0)).any()


def test_class_agnostic_nms_vs_greedy_reference():
    import unicorn_oracle as orc
    from test_det import agnostic_reference
    from unicorn_b200 import ops, post_ops
    g = torch.Generator().manual_seed(3)
    A, ncls = 3000, 80
    pred = torch.zeros(A, 5 + ncls)
    ctr = torch.rand(40, 2, generator=g) * 600 + 50  # 40 clusters of overlapping boxes of random classes
    idx = torch.randint(0, 40, (A,), generator=g)
    pred[:, :2] = ctr[idx] + torch.randn(A, 2, generator=g) * 6
    pred[:, 2:4] = 40 + torch.rand(A, 2, generator=g) * 30
    pred[:, 4] = torch.rand(A, generator=g)
    pred[:, 5:] = torch.rand(A, ncls, generator=g) * 0.5
    pred[torch.arange(A), 5 + torch.randint(0, ncls, (A,), generator=g)] = 0.5 + torch.rand(A, generator=g) * 0.5
    ws = ops.PostWorkspace(A, "cuda")
    for conf, thr in ((0.01, 0.3), (0.2, 0.65)):
        d, cnt = post_ops.postprocess_device_ex(pred.cuda(), ncls, conf, thr, ws, class_agnostic=True)
        n = int(cnt.item())
        ref = agnostic_reference(orc, pred, conf, thr)
        assert n == ref.shape[0] and n < 0.5 * (pred[:, 4] * pred[:, 5:].max(1)[0] >= conf).sum()
        assert torch.equal(d[:n].cpu(), ref)
        # the class-aware mode of the new entry point is the existing postprocess
        ws2 = ops.PostWorkspace(A, "cuda")
        d1, c1 = post_ops.postprocess_device_ex(pred.cuda(), ncls, conf, thr, ws)
        d2, c2 = ops.postprocess_device(pred.cuda(), ncls, conf, thr, ws2)
        n1 = int(c1.item())
        assert n1 == int(c2.item()) > n and torch.equal(d1[:n1], d2[:n1])


@pytest.fixture(scope="module")
def det_engine():
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.weights import make_state_dict
    return UnicornEngine(make_state_dict("unicorn_det_convnext_tiny", 0), "unicorn_det_convnext_tiny")


def test_det_engine_rejects_tracking_stages(det_engine):
    e = det_engine
    x = torch.zeros(1, 20, 20, 384, dtype=torch.bfloat16, device="cuda")
    for call in (lambda: e.interaction(x, x), lambda: e.upsample(x, "t"), lambda: e.propagate(x, x, None), lambda: e.mask_branch([x] * 3),
                 lambda: e.project_ref(x), lambda: e.head([x] * 3, None, "sot")):
        with pytest.raises(ValueError, match="detector"):
            call()


def test_detector_partial_batches_mixed_sizes_graph_and_eager(det_engine):
    from unicorn_b200.det import UnicornDetector
    from unicorn_b200.synthetic import make_video
    frames, _ = make_video(3, 480, 640, seed=5, n_obj=4)
    bgr = frames.permute(0, 2, 3, 1).clamp(0, 255).to(torch.uint8).numpy()
    images = [bgr[0], np.ascontiguousarray(bgr[1][:300, :500]), np.ascontiguousarray(bgr[2][:200])]
    size = (416, 640)
    one = UnicornDetector(det_engine, size, max_batch=1)
    solo = [one.detect([im])[0] for im in images]
    solo2 = [one.detect([im])[0] for im in images]  # replays of the captured graph
    assert all(a[1] == b[1] and torch.equal(a[0], b[0]) for a, b in zip(solo, solo2))
    assert all(r.shape[0] > 0 for r, _ in solo)
    for use_graph in (True, False):
        det = UnicornDetector(det_engine, size, max_batch=4, use_graph=use_graph)
        for batch in (images, images[1:], images[:1]):  # partial batches of the 4-image graph
            out = det.detect(batch)
            want = solo if batch is images else solo[1:] if len(batch) == 2 else solo[:1]
            for (r, s), (rw, sw) in zip(out, want):
                assert s == sw and torch.equal(r, rw), (r.shape, rw.shape)
    # RGB input: the same rows as its BGR original
    rgb = one.detect([np.ascontiguousarray(images[0][..., ::-1])], rgb=True)[0]
    assert torch.equal(rgb[0], solo[0][0])
    # two steps in flight
    det = UnicornDetector(det_engine, size, max_batch=2, depth=2)
    det.submit(images[:2])
    det.submit(images[2:])
    a, b = det.collect(), det.collect()
    assert torch.equal(a[0][0], solo[0][0]) and torch.equal(a[1][0], solo[1][0]) and torch.equal(b[0][0], solo[2][0])

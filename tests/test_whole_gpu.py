"""`mode="whole"` (SURVEY §8 a13: unicorn/models/unicorn.py:133-139 — zero priors, MOT prediction set) on the H100 engine against
the outputs of the UNMODIFIED reference (tests/golden/whole_tiny_320.npz, written by tests/golden/make_golden_whole.py), for the
plain model (MOT detector) and the mask model (MOTS detector: controllers + mask branch).

Tolerances are those of tests/test_engine_gpu.py (bf16 operands vs the reference's fp32): probabilities 5e-2 abs, box centre 0.2
grid cells, log(w,h) 0.2, dynamic-conv parameters / mask features 8e-2 of the tensor's max."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

STRIDE_ROWS = torch.cat([torch.full((n,), float(s)) for n, s in ((1600, 8), (400, 16), (100, 32))])


def rel(a, b):
    a, b = a.float().cpu(), torch.as_tensor(b).float()
    return ((a - b).abs().max() / (b.abs().max() + 1e-12)).item()


@pytest.fixture(scope="module")
def golden():
    from unicorn_b200.synthetic import make_video
    g = np.load(os.path.join(ROOT, "tests", "golden", "whole_tiny_320.npz"))
    frames, _ = make_video(2, 320, 320, seed=int(g["seed_video"]), n_obj=int(g["n_obj"]))
    f = int(g["frame"])
    return g, frames[f:f + 1].cuda()


def check_head(head, href):
    head, href = head.float().cpu(), torch.as_tensor(href)
    assert head.shape == href.shape
    errs = dict(xy=((head[0, :, :2] - href[0, :, :2]).abs().max(dim=1)[0] / STRIDE_ROWS).max().item(),
                logwh=(torch.log(head[0, :, 2:4]) - torch.log(href[0, :, 2:4])).abs().max().item(),
                score=(head[..., 4:] - href[..., 4:]).abs().max().item())
    print("whole-mode head errors vs the reference golden:", errs)
    assert errs["xy"] < 0.2 and errs["logwh"] < 0.2 and errs["score"] < 5e-2, errs


def check_dets(dets, ref, orc):
    """same decisions up to threshold flips: counts within 5 %, every engine detection is a reference detection (same class,
    IoU > 0.7, score within 5e-2)"""
    ref = torch.as_tensor(ref)
    n = dets.shape[0]
    assert abs(n - ref.shape[0]) <= max(5, 0.05 * ref.shape[0]), (n, ref.shape[0])
    iou = orc.box_iou_np(dets[:, :4].numpy(), ref[:, :4].numpy())
    iou[dets[:, 6].numpy()[:, None] != ref[:, 6].numpy()[None, :]] = 0.0  # class aware
    j = iou.argmax(1)
    strong = (dets[:, 4] * dets[:, 5]).numpy() > 0.05  # rows far from the confidence threshold must all be matched
    assert (iou.max(1)[strong] > 0.7).all(), iou.max(1)[strong]
    sc, sr = (dets[:, 4] * dets[:, 5]).numpy(), (ref[:, 4] * ref[:, 5]).numpy()[j]
    assert np.abs(sc - sr)[iou.max(1) > 0.7].max() < 5e-2


def test_mot_mode_head_and_detections_vs_reference_golden(golden):
    import unicorn_oracle as orc
    from unicorn_b200 import ops
    from unicorn_b200.compat.model import UnicornB200Model, postprocess
    from unicorn_b200.weights import make_state_dict
    g, img = golden
    model = UnicornB200Model(make_state_dict("unicorn_track_tiny", 0), "unicorn_track_tiny").eval()
    head, seq = model(imgs=img, mode="whole")
    assert rel(seq["feat"][0, ::4], g["feat_sub"]) < 4e-2
    check_head(head, g["head"])
    head_cxcywh = head.clone()
    dets = postprocess(head, 8, float(g["conf"]), float(g["nms"]))[0]  # like the reference's, it turns head's boxes into corners in place
    assert dets is not None and torch.allclose(head[0, :, 2] - head[0, :, 0], head_cxcywh[0, :, 2], atol=1e-3)
    head = head_cxcywh
    check_dets(dets.cpu(), g["dets"], orc)
    # the MOT driver's device half gives the same head output, bit for bit (same kernels, other buffers)
    from unicorn_b200.mot import UnicornMOTTracker
    trk = UnicornMOTTracker(model.engine, (320, 320), conf=float(g["conf"]), nms=float(g["nms"]))
    trk.step_tensor(img)
    assert torch.equal(trk.last["head"], head), (trk.last["head"] - head).abs().max()
    # exact decisions on the reference's own head output (NMS kernels, 8 classes)
    ws = ops.PostWorkspace(2100, "cuda")
    d, cnt = ops.postprocess_device(torch.from_numpy(g["head"]).cuda()[0].contiguous(), 8, float(g["conf"]), float(g["nms"]), ws)
    n = int(cnt.item())
    ref = torch.from_numpy(g["dets"])
    assert n == ref.shape[0]
    got = d[:n].cpu()
    assert torch.cdist(got[:, :6], ref[:, :6], p=float("inf")).min(dim=0)[0].max().item() < 1e-4
    assert torch.equal(got[:, 6].sort()[0], ref[:, 6].sort()[0])


def test_mask_model_whole_mode_vs_reference_golden(golden):
    import unicorn_oracle as orc
    from unicorn_b200 import ops
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.weights import make_state_dict
    g, img = golden
    name = "unicorn_track_tiny_mask"
    e = UnicornEngine(make_state_dict(name, 0), name)
    e.begin_frame()
    fpn, _ = e.backbone(img, tag="t")
    head = e.head(fpn, None, "mot", with_masks=True)
    check_head(head, g["m_head"])
    dyn = torch.cat([d[0, :, :, :169].reshape(-1, 169) for d in e.dyn_levels], 0)
    assert rel(dyn[::16], g["m_dyn_sub"]) < 8e-2
    mf, um = e.mask_branch(fpn)
    assert rel(mf.permute(0, 3, 1, 2), g["m_mask_feats"]) < 8e-2
    assert rel(um.permute(0, 3, 1, 2)[0, :, ::4, ::4], g["m_up_masks_sub"]) < 8e-2
    ws = ops.PostWorkspace(2100, "cuda")
    dets, cnt = ops.postprocess_device(head[0], 8, float(g["conf"]), float(g["nms"]), ws)
    n = int(cnt.item())
    check_dets(dets[:n].cpu(), g["m_dets"], orc)
    # masks of the top instances: the engine's top detection is the reference's top detection and their masks agree
    hw = [(t.shape[1], t.shape[2]) for t in e.dyn_levels]
    masks = ops.dynamic_masks(mf, um, e.dyn_levels, hw, ws, int(g["keep"]), up_rate=4, d_rate=2)
    ref = torch.from_numpy(g["m_dets"])
    iou = orc.box_iou_np(dets[:1, :4].cpu().numpy(), ref[:int(g["keep"]), :4].numpy())
    print("top detection IoU with the reference's top instances:", iou)
    assert iou.max() > 0.7  # measured 0.81: log(w,h) of the bf16 head is within 0.15 of the reference's
    if iou.argmax() == 0 and iou.max() > 0.9:
        m, r = masks[0].cpu()[::2, ::2], torch.from_numpy(g["m_mask0_sub"].astype(np.float32))
        mb, rb = m > 0.3, r > 0.3
        inter, union = (mb & rb).sum().item(), (mb | rb).sum().item()
        print("top-instance mask IoU vs the reference golden (bf16 features):", inter / max(union, 1))
        assert union == 0 or inter / union > 0.9

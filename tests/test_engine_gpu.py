"""End-to-end parity of the CUDA engine against the CPU oracle and the golden fixtures (tiny 320x320 SOT frame).

Tolerances (relative to each tensor's max magnitude; the engine computes in bf16 operands / fp32 accumulate, the
oracle in fp32): neck maps 8e-2, backbone feat 4e-2, interaction / embeddings 5e-2, propagated prior 6e-2 abs,
head: box centre 0.2 grid cells, log(w,h) 0.2, obj/cls probabilities 5e-2 abs."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).abs().max() / (b.abs().max() + 1e-12)).item()


def nchw(t):
    return t.float().permute(0, 3, 1, 2).cpu()


@pytest.fixture(scope="module")
def setup():
    import unicorn_oracle as orc
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.sot import UnicornSOTTrack
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.weights import make_state_dict
    name = "unicorn_track_tiny"
    sd = make_state_dict(name, 0)
    frames, boxes = make_video(3, 320, 320, seed=0)
    o = orc.SOTOracle(sd, name)
    o.initialize(frames[0:1], boxes[0, 0])
    st = {}
    o.track(frames[2:3], st)
    eng = UnicornEngine(sd, name)
    trk = UnicornSOTTrack(eng, (320, 320), use_graph=False, full_nms=True)
    trk.initialize_tensor(frames[0:1], boxes[0, 0])
    dets, n = trk.track_tensor(frames[2:3])
    torch.cuda.synchronize()
    return dict(st=st, trk=trk, dets=dets, n=n, frames=frames, boxes=boxes, sd=sd, orc=orc)


def test_stage_parity_vs_oracle(setup):
    st, last = setup["st"], setup["trk"].last
    errs = {}
    for i in range(3):
        errs[f"fpn{i}"] = rel(nchw(last["fpn"][i]), st["fpn"][i])
    errs["feat"] = rel(nchw(last["feat"]), st["feat"])
    errs["inter_pre"] = rel(nchw(last["inter_pre"]), st["inter_pre"])
    errs["inter_cur"] = rel(nchw(last["inter_cur"]), st["inter_cur"])
    errs["embed_pre"] = rel(nchw(last["embed_pre"]), st["embed_pre"])
    errs["embed_cur"] = rel(nchw(last["embed_cur"]), st["embed_cur"])
    errs["coarse"] = (last["priors"][0].cpu() - st["coarse"][0]).abs().max().item()
    head, href = last["head"].cpu(), st["head"]
    stride = torch.cat([torch.full((n,), float(s)) for n, s in ((1600, 8), (400, 16), (100, 32))])
    errs["head_xy"] = ((head[0, :, :2] - href[0, :, :2]).abs().max(dim=1)[0] / stride).max().item()  # in cells
    errs["head_logwh"] = (torch.log(head[0, :, 2:4]) - torch.log(href[0, :, 2:4])).abs().max().item()
    errs["head_score"] = (head[..., 4:] - href[..., 4:]).abs().max().item()
    print("stage errors:", {k: f"{v:.3e}" for k, v in errs.items()})
    tol = dict(fpn0=8e-2, fpn1=8e-2, fpn2=8e-2, feat=4e-2, inter_pre=5e-2, inter_cur=5e-2, embed_pre=5e-2, embed_cur=5e-2,
               coarse=6e-2, head_xy=0.2, head_logwh=0.2, head_score=5e-2)
    bad = {k: v for k, v in errs.items() if not v <= tol[k]}
    assert not bad, f"out of tolerance: {bad} (all: {errs})"


def test_golden_fixture(setup):
    g = np.load(os.path.join(ROOT, "tests", "golden", "sot_tiny_320.npz"))
    last = setup["trk"].last
    assert rel(nchw(last["fpn"][2])[0, ::4], torch.from_numpy(g["fpn2"])) < 8e-2
    assert rel(nchw(last["embed_cur"])[0, :, ::4, ::4], torch.from_numpy(g["embed_cur_sub"])) < 5e-2
    assert (last["priors"][0].cpu() - torch.from_numpy(g["coarse"])[0]).abs().max().item() < 6e-2
    assert (last["head"].cpu()[..., 4:] - torch.from_numpy(g["head"])[..., 4:]).abs().max().item() < 5e-2


def test_detections_vs_oracle(setup):
    """NMS runs on slightly different scores, so compare decisions robustly: the top detection must match a top-3
    oracle detection (IoU > 0.9) and the kept counts must be close."""
    orc = setup["orc"]
    dets, n = setup["dets"], setup["n"]
    ref = setup["st"]["dets"]
    assert n > 0 and ref is not None
    assert abs(n - ref.shape[0]) <= max(5, 0.05 * ref.shape[0]), (n, ref.shape[0])
    # every reported top detection must exist in the oracle's list: same box (IoU > 0.7) with score within 3e-2
    iou = orc.box_iou_np(dets[:, :4].numpy(), ref[:, :4].numpy())
    j = iou.argmax(1)
    assert (iou.max(1) > 0.7).all(), iou.max(1)
    sc = (dets[:, 4] * dets[:, 5]).numpy()
    sr = (ref[:, 4] * ref[:, 5]).numpy()[j]
    assert np.abs(sc - sr).max() < 5e-2, (sc, sr)


def test_postprocess_exact_on_oracle_head(setup):
    """Device NMS on the oracle's own head output must reproduce the oracle's detections exactly (bit-level decisions)."""
    from unicorn_b200 import ops
    orc = setup["orc"]
    head = setup["st"]["head"].cuda().contiguous()
    ws = ops.PostWorkspace(head.shape[1], "cuda")
    dets, cnt = ops.postprocess_device(head[0], 1, 0.001, 0.65, ws)
    n = int(cnt.item())
    ref = setup["st"]["dets"]
    assert n == ref.shape[0]
    assert torch.allclose(dets[:n].cpu(), ref, rtol=0, atol=1e-5)


def test_cuda_graph_replay_matches_eager(setup):
    from unicorn_b200.sot import UnicornSOTTrack
    trk = setup["trk"]
    frames, boxes = setup["frames"], setup["boxes"]
    g = UnicornSOTTrack(trk.eng, (320, 320), use_graph=True)
    g.initialize_tensor(frames[0:1], boxes[0, 0])
    d1, n1 = g.track_tensor(frames[1:2].pin_memory())
    d2, n2 = g.track_tensor(frames[2:3].pin_memory())
    # every kernel is deterministic (GroupNorm statistics use integer atomics): graph replay == eager, bit for bit
    # the graph tracker stops NMS after max_inst kept boxes: its rows are exactly the head of the full result
    assert n2 == min(setup["n"], 3), (n2, setup["n"])
    assert torch.equal(d2, setup["dets"][:n2]), (d2, setup["dets"])


def test_reference_api_facade(setup):
    """unicorn_b200.compat.model: the reference's stage-by-stage calling convention (unicorn_sot.py:78-109 written out with
    model(..., mode=...) calls, NCHW fp32 tensors and the plain torch mm + softmax(dim=0) correlation of the reference) on
    the H100 engine; same tolerances as the fused driver, and seq_dict must survive copy.deepcopy (mot_evaluator.py:1015)."""
    import copy
    import torch.nn.functional as F
    from unicorn_b200.compat.model import UnicornB200Model, postprocess
    from unicorn_b200.sot import get_label_map
    st, frames, boxes = setup["st"], setup["frames"], setup["boxes"]
    model = UnicornB200Model(setup["sd"], "unicorn_track_tiny").eval()
    ref_img, cur_img = frames[0:1].cuda(), frames[2:3].cuda()
    _, d0 = model(imgs=ref_img, mode="backbone")
    d0 = copy.deepcopy(d0)
    fpn, d1 = model(imgs=cur_img, mode="backbone")
    assert set(d1) == {"feat", "pos", "h", "w"} and rel(d1["pos"], st["pos"]) < 1e-3
    f0, f1 = model(seq_dict0=d0, seq_dict1=d1, mode="interaction")
    e0, e1 = model(feat=f0, mode="upsample"), model(feat=f1, mode="upsample")
    assert rel(f1, st["inter_cur"]) < 5e-2 and rel(e1, st["embed_cur"]) < 5e-2
    for i in range(3):
        assert rel(fpn[i], st["fpn"][i]) < 8e-2
    lbl = F.interpolate(get_label_map(boxes[0, 0], 320, 320, "cuda"), scale_factor=1 / 8, mode="bilinear", align_corners=False)
    k, q = e0.half().flatten(-2)[0], e1.half().flatten(-2)[0]          # (C, N) each — unicorn_sot.py:92-97
    trans = torch.softmax(torch.mm(k.t(), q).float(), dim=0)           # softmax over the reference positions
    coarse = torch.mm(lbl.view(1, -1).float(), trans).view(1, 1, 40, 40)
    assert (coarse[0].cpu() - st["coarse"][0]).abs().max().item() < 6e-2
    pri = [coarse, F.interpolate(coarse, scale_factor=1 / 2, mode="bilinear", align_corners=False),
           F.interpolate(coarse, scale_factor=1 / 4, mode="bilinear", align_corners=False)]
    out = model.head(fpn, pri, mode="sot")
    assert out.shape == st["head"].shape
    assert (out.cpu()[..., 4:] - st["head"][..., 4:]).abs().max().item() < 5e-2
    dets = postprocess(out, 1, 0.001, 0.65)[0]
    assert dets is not None and abs(dets.shape[0] - st["dets"].shape[0]) <= max(5, 0.05 * st["dets"].shape[0])
    whole, _ = model(imgs=cur_img, mode="whole")
    assert whole.shape == (1, 2100, 5 + model.num_classes)
    with pytest.raises(ValueError):
        model(imgs=cur_img, mode="train")


def test_pipelined_tracker_matches_sequential(setup):
    """depth=2: two frames in flight on two streams / engine contexts (sot.py submit / collect).  The frames of a sequence are
    independent, so every result must equal the sequential tracker's, bit for bit, in order.  Then the same for two sequences per
    step (n_seq = 2)."""
    from unicorn_b200.sot import UnicornSOTBatch, UnicornSOTTrack
    from unicorn_b200.synthetic import make_video
    trk = setup["trk"]
    frames, boxes = make_video(8, 320, 320, seed=6)
    host = [frames[i:i + 1].pin_memory() for i in range(8)]
    seq = UnicornSOTTrack(trk.eng, (320, 320), use_graph=True)
    seq.initialize_tensor(host[0], boxes[0, 0])
    ref = [seq.track_tensor(host[i]) for i in range(1, 8)]
    pipe = UnicornSOTTrack(trk.eng, (320, 320), use_graph=True, depth=2)
    pipe.initialize_tensor(host[0], boxes[0, 0])
    got = []
    pipe.submit(host[1])
    for i in range(2, 8):
        pipe.submit(host[i])
        got.append(pipe.collect())
    got.append(pipe.collect())
    for (d0, n0), (d1, n1) in zip(ref, got):
        assert n0 == n1 and torch.equal(d0, d1)
    # the synchronous call of a pipelined tracker is submit + collect
    d, n = pipe.track_tensor(host[3])
    assert n == ref[2][1] and torch.equal(d, ref[2][0])
    # n_seq = 2: the second sequence is another video, its frames fed in reverse order
    frames2, boxes2 = make_video(8, 320, 320, seed=7)
    steps = [torch.stack([frames[i], frames2[8 - i]]).pin_memory() for i in range(1, 8)]
    seq2 = UnicornSOTBatch(trk.eng, (320, 320), 2, use_graph=True)
    pipe2 = UnicornSOTBatch(trk.eng, (320, 320), 2, use_graph=True, depth=2)
    for b in (seq2, pipe2):
        b.initialize_tensor(0, host[0], boxes[0, 0])
        b.initialize_tensor(1, frames2[0:1], boxes2[0, 0])
    ref2 = [seq2.track_tensor(s) for s in steps]
    pipe2.submit(steps[0])
    got2 = []
    for s in steps[1:]:
        pipe2.submit(s)
        got2.append(pipe2.collect())
    got2.append(pipe2.collect())
    assert all(c.graph is not None for c in pipe2._ctxs)
    for t, ((d0, n0), (d1, n1)) in enumerate(zip(ref2, got2)):
        assert torch.equal(n0, n1), f"step {t}"
        for i in range(2):
            k = min(int(n0[i]), 3)
            assert torch.equal(d0[i, :k], d1[i, :k]), f"step {t} sequence {i}"

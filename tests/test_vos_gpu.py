"""VOS driver (unicorn_b200/vos.py) against the label maps of the UNMODIFIED reference class UnicornVOSTrack
(tests/golden/vos_tiny.npz: two first-frame objects, a third appearing in frame 2, soft aggregation, mask resize to the original
frame) and the device-side result assembly (uc_vos_aggregate) against its torch / numpy definition."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))


def test_vos_aggregate_kernel_matches_definition():
    """unicorn_vos.py:139-155 (F.interpolate(scale_factor=1/r)[:H,:W] into a zero map) + :105-121 (float32 background product in
    list order, argmax with the lower channel winning ties) on random soft masks, one object given by its initial label map."""
    from unicorn_b200 import ops
    g = torch.Generator().manual_seed(3)
    Hin, Win, H0, W0 = 96, 160, 113, 187
    r = min(Hin / H0, Win / W0)
    ids = [4, 1, 7, 2]  # list order != id order: the product follows the list, ties go to the lower id
    masks = torch.rand(3, Hin, Win, generator=g)
    masks[0, :40] = 1.0   # saturated region: background product is exactly 0 there
    masks[1, :20] = 1.0   # ... and two objects tie at 1.0
    lab = torch.zeros(H0, W0, dtype=torch.uint8)
    lab[30:70, 50:120] = 2
    soft_ref = np.zeros((4, H0, W0), dtype=np.float32)
    m = F.interpolate(masks[:, None], scale_factor=1 / r, mode="bilinear", align_corners=False)[:, 0, :H0, :W0]
    soft_ref[:3, :m.shape[1], :m.shape[2]] = m.numpy()
    soft_ref[3] = (lab.numpy() == 2)
    merge = np.zeros((H0, W0, 8))
    for k, i in enumerate(ids):
        merge[:, :, i] = soft_ref[k]
    merge[:, :, 0] = np.prod(1 - np.stack(list(soft_ref), -1), axis=-1)
    seg_ref = np.argmax(merge, -1).astype(np.uint8)
    md, ld = masks.cuda().contiguous(), lab.cuda()
    soft = torch.zeros(4, H0, W0, device="cuda")
    seg = torch.zeros(H0, W0, dtype=torch.uint8, device="cuda")
    ops.vos_aggregate([md[k] for k in range(3)], ld, ids, Hin, Win, r, soft, seg)
    assert np.abs(soft.cpu().numpy() - soft_ref).max() < 2e-6
    agree = (seg.cpu().numpy() == seg_ref).mean()
    assert agree > 0.9995, agree  # exact up to last-ulp differences of the bilinear weights at near ties


def _run_driver(use_graph, keep_soft=False):
    from make_golden_vos_common import make_sequence
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.vos import UnicornVOSTrack
    from unicorn_b200.weights import make_state_dict
    g = np.load(os.path.join(ROOT, "tests", "golden", "vos_tiny.npz"))
    name, size, new_at = str(g["config"]), tuple(int(v) for v in g["size"]), int(g["new_at"])
    rgb, xywh, lab = make_sequence()
    trk = UnicornVOSTrack(UnicornEngine(make_state_dict(name, 0), name), size, use_graph=use_graph)
    trk.debug = keep_soft  # keep a copy of every object's head output (the score margins of the parity test)
    trk.initialize(rgb[0], {"init_object_ids": ["1", "2"], "sequence_object_ids": ["1", "2", "3"],
                            "init_bbox": {"1": xywh[0, 0].tolist(), "2": xywh[0, 1].tolist()}})
    segs, states, softs = [], [], []
    for t in range(1, int(g["n_frames"])):
        info = {"init_object_ids": ["3"], "init_bbox": {"3": xywh[t, 2].tolist()}, "init_mask": lab} if t == new_at else {}
        n_obj = len(trk.obj_ids) + (1 if t == new_at else 0)
        segs.append(trk.track(rgb[t], info)["segmentation"].copy())
        states.append([trk.state_pre_dict[o] for o in ("1", "2")])
        if keep_soft:
            heads = {o: po["head"].float().cpu() for o, po in trk.last["per_obj"].items()}
            softs.append((trk._soft[:n_obj].cpu().numpy().copy(), heads))
    return g, segs, states, softs


def _oracle_softs(g):
    """fp32 oracle of the same sequence: per frame (label map, soft masks in list order) — the decision margins come from here."""
    import unicorn_oracle as orc
    from make_golden_vos_common import box_xyxy, make_sequence, prep_frame
    from unicorn_b200.weights import make_state_dict
    name, size = str(g["config"]), tuple(int(v) for v in g["size"])
    H0, W0, new_at = int(g["H0"]), int(g["W0"]), int(g["new_at"])
    rgb, xywh, lab = make_sequence()
    r = min(size[0] / H0, size[1] / W0)
    o = orc.VOSOracle(make_state_dict(name, 0), name, half_corr=True)
    o.initialize(prep_frame(rgb[0], size), {"1": box_xyxy(xywh[0, 0], r), "2": box_xyxy(xywh[0, 1], r)}, orig_size=(H0, W0), r=r)
    out = []
    for t in range(1, int(g["n_frames"])):
        new = {"3": box_xyxy(xywh[t, 2], r)} if t == new_at else None
        seg, res = o.track(prep_frame(rgb[t], size), new, lab if t == new_at else None)
        ids = ["1", "2"] + (["3"] if t >= new_at else [])
        out.append((seg, np.stack([np.asarray(res[i]["soft"], dtype=np.float32) for i in ids]),
                    {i: res[i]["head"] for i in ids if res[i].get("head") is not None}))
    return out


def _top1_margin(head):
    """head [1,N,6] (cx, cy, w, h, obj, cls): (corner box of the best-scoring anchor, its score lead over the best anchor that
    is a DIFFERENT instance (IoU < 0.5 with it), all scores)."""
    import unicorn_oracle as orc
    h = head[0].float()
    sc = h[:, 4] * h[:, 5]
    b = torch.stack([h[:, 0] - h[:, 2] / 2, h[:, 1] - h[:, 3] / 2, h[:, 0] + h[:, 2] / 2, h[:, 1] + h[:, 3] / 2], 1)
    k = int(sc.argmax())
    iou = torch.from_numpy(orc.box_iou_np(b[k:k + 1].numpy(), b.numpy())[0])
    other = sc[iou < 0.5]
    return b[k], float(sc[k] - (other.max() if other.numel() else 0.0)), sc


def test_vos_driver_vs_reference_class_golden():
    """Label maps of the product driver (reference protocol: RGB frames in, `segmentation` out) against the UNMODIFIED reference
    class's.  Two decisions feed a pixel's label, and with seeded random weights both are near ties, so both are compared margin aware:
      * per object, WHICH instance gets the mask (top-1 of obj * cls after NMS, unicorn_vos.py:137-155).  It is well conditioned when
        the fp32 oracle's best anchor leads every different instance by more than twice the largest score error of the engine on that
        object: then the engine must pick the same instance, and wherever both picked the same instance (conditioned or not) its soft
        mask must stay within SOFT_TOL of the oracle's.  Picks of another instance on an ill-conditioned object are counted and reported;
      * per pixel, the argmax over the soft masks: where the oracle's winning channel leads by more than MARGIN the engine must agree
        (>= 99 %); the raw agreement is reported and bounded on the frames without an instance flip."""
    import unicorn_oracle as orc
    MARGIN, SOFT_TOL = 0.12, 0.12  # measured soft-mask drift p99 <= 0.036: the margin is > 3x that
    g, segs, states, softs = _run_driver(False, keep_soft=True)
    orc_frames = _oracle_softs(g)
    new_at = int(g["new_at"])
    report = dict(raw_agreement=[], conditioned_agreement=[], conditioned_fraction=[], soft_err_p99=[], oracle_vs_reference=[],
                  instance_flips=[], well_conditioned_objects=0, objects=0)
    for t, (s, r) in enumerate(zip(segs, g["segs"])):
        o_seg, o_soft, o_heads = orc_frames[t]
        e_soft, e_heads = softs[t]
        ids = ["1", "2"] + (["3"] if t + 1 >= new_at else [])
        same = []
        for k, oid in enumerate(ids):
            if oid not in o_heads or oid not in e_heads:  # the frame where the object appears: its mask is the given label map
                same.append(k)
                continue
            ob, margin, osc = _top1_margin(o_heads[oid])
            eb, _, esc = _top1_margin(e_heads[oid])
            eps = float((osc - esc).abs().max())
            agree = orc.box_iou_np(ob[None].numpy(), eb[None].numpy())[0, 0] > 0.5
            report["objects"] += 1
            if margin > 2 * eps:
                report["well_conditioned_objects"] += 1
                assert agree, (t, oid, margin, eps)
            if agree:
                same.append(k)
            else:
                report["instance_flips"].append((t, oid, margin, eps))
        chans = np.concatenate([np.prod(1 - o_soft, axis=0, keepdims=True), o_soft], 0)
        top2 = np.sort(chans, axis=0)[-2:]
        cond = (top2[1] - top2[0]) > MARGIN
        if len(same) == len(ids):
            report["raw_agreement"].append(float((s == r).mean()))
            report["conditioned_agreement"].append(float((s == r)[cond].mean()) if cond.any() else 1.0)
        report["conditioned_fraction"].append(float(cond.mean()))
        report["oracle_vs_reference"].append(float((o_seg == r).mean()))
        report["soft_err_p99"].append(float(np.percentile(np.abs(e_soft[same] - o_soft[same]), 99)) if same else 0.0)
    print("VOS driver vs the reference class:", report)
    out = os.environ.get("UC_REPORT_DIR", "")  # optional directory for the measured parity reports
    if os.path.isdir(out):
        import json
        json.dump(report, open(os.path.join(out, "r2_vos_parity.json"), "w"), indent=1)
    assert len(report["instance_flips"]) <= 2 and len(report["raw_agreement"]) >= 2, report
    assert min(report["conditioned_agreement"]) > 0.99, report
    assert min(report["raw_agreement"]) > 0.8, report
    assert max(report["soft_err_p99"]) < SOFT_TOL, report
    assert segs[new_at - 1].max() == 3  # the new object's initial mask went through the aggregation
    print("max |state box - reference| (pixels):", np.abs(np.array(states, dtype=np.float32) - g["states"]).max())


def test_vos_graph_replay_matches_eager():
    _, segs_e, st_e, _ = _run_driver(False)
    _, segs_g, st_g, _ = _run_driver(True)
    for a, b in zip(segs_e, segs_g):
        assert np.array_equal(a, b)
    assert st_e == st_g


def test_vos_three_frames_in_flight_match_sequential():
    """submit / collect with depth=3 (worker drivers on engine forks, own streams, CUDA graphs): label maps, soft masks and detection
    rows of every frame are bit-identical to the synchronous driver's; a frame that adds an object drains the pipeline and the
    workers pick the new reference group up."""
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.vos import UnicornVOSTrack
    from unicorn_b200.weights import make_state_dict
    name = "unicorn_track_tiny_mask"
    eng = UnicornEngine(make_state_dict(name, 0), name)
    frames, boxes = make_video(12, 320, 320, seed=9, n_obj=3)
    u8 = frames.round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()
    lab = torch.zeros(320, 320, dtype=torch.uint8)
    x1, y1, x2, y2 = boxes[6, 2].int().tolist()
    lab[y1:y2, x1:x2] = 3

    def run(depth):
        trk = UnicornVOSTrack(eng, (320, 320), use_graph=True, depth=depth)
        trk.initialize_tensor(u8[0:1], {1: boxes[0, 0], 2: boxes[0, 1]})
        out = []

        def keep(o):
            out.append((o["segmentation"].cpu().clone(), o["soft"].cpu().clone(), {k: (None if v[0] is None else v[0].clone()) for k, v in o["objects"].items()}))
        order = list(range(1, 6))
        if depth == 1:
            for t in order:
                keep(trk.track_tensor(u8[t:t + 1]))
        else:
            sub = 0
            for k in range(len(order)):
                while sub < len(order) and sub - k < depth:
                    trk.submit(u8[order[sub]:order[sub] + 1].pin_memory())
                    sub += 1
                keep(trk.collect())
        keep(trk.track_tensor(u8[6:7], {3: boxes[6, 2]}, lab))  # object 3 appears: synchronous path, pipeline drained
        order = list(range(7, 12))
        if depth == 1:
            for t in order:
                keep(trk.track_tensor(u8[t:t + 1]))
        else:
            sub = 0
            for k in range(len(order)):
                while sub < len(order) and sub - k < depth:
                    trk.submit(u8[order[sub]:order[sub] + 1].pin_memory())
                    sub += 1
                keep(trk.collect())
        return out
    ref, got = run(1), run(3)
    assert len(ref) == len(got) == 11 and got[-1][1].shape[0] == 3
    for t, (r, g) in enumerate(zip(ref, got)):
        assert torch.equal(r[0], g[0]) and torch.equal(r[1], g[1]), f"frame {t}"
        assert r[2].keys() == g[2].keys()
        for k in r[2]:
            assert (r[2][k] is None) == (g[2][k] is None) and (r[2][k] is None or torch.equal(r[2][k], g[2][k])), (t, k)

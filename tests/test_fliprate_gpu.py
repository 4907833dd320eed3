"""End-to-end decision parity over a sequence (SURVEY §7 "report flip rate"; north_star "bit-matching track assignments"):
the bf16 engine and the fp32 oracle run the SAME 32-frame synthetic video, each on its own detections, and the decisions
are compared frame by frame.

  * SOT (unicorn_sot.py:57-77): the top-1 box after NMS.  A frame "flips" when the engine's box is not the oracle's box
    (IoU < 0.5).  With seeded random weights the best scores are nearly tied (0.0120 / 0.0115 / 0.0111 ...), so a flip is only a
    defect when the decision is well conditioned: oracle margin s1 - s2 larger than twice the largest score error the engine
    makes on that frame.  Bound: NO flip among well-conditioned frames; the overall rate is reported.
  * MOT (mot_evaluator.py:1005-1057 + QuasiDenseEmbedTracker): (a) ids from engine embeddings vs oracle embeddings on identical
    boxes must match bit for bit; (b) the raw end-to-end id-flip count (each side on its own detections; tracks paired by box
    IoU > 0.7, first pairing fixes the id map, later disagreements are flips) is reported.

The measured rates are printed and, if UC_REPORT_DIR names a directory, written to it as r2_fliprate.json."""
import json
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
N_FRAMES = 32
REPORT = {}


def _save():
    out = os.environ.get("UC_REPORT_DIR", "")  # optional directory for the measured parity reports
    if os.path.isdir(out):
        json.dump(REPORT, open(os.path.join(out, "r2_fliprate.json"), "w"), indent=1)


def test_sot_top1_flip_rate():
    import unicorn_oracle as orc
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.sot import UnicornSOTTrack
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.weights import make_state_dict
    name = "unicorn_track_tiny"
    sd = make_state_dict(name, 0)
    frames, boxes = make_video(N_FRAMES, 320, 320, seed=3)
    o = orc.SOTOracle(sd, name)
    o.initialize(frames[0:1], boxes[0, 0])
    trk = UnicornSOTTrack(UnicornEngine(sd, name), (320, 320), use_graph=True, max_inst=3)
    trk.initialize_tensor(frames[0:1], boxes[0, 0])
    flips, hard_flips, well, ious, eps_all = 0, 0, 0, [], []
    for t in range(1, N_FRAMES):
        st = {}
        ref = o.track(frames[t:t + 1], st)
        dets, n = trk.track_tensor(frames[t:t + 1].pin_memory())
        assert n > 0 and ref is not None
        so = (st["head"][0, :, 4] * st["head"][0, :, 5])
        se = (trk.last["head"][0, :, 4] * trk.last["head"][0, :, 5]).cpu()
        eps = (so - se).abs().max().item()
        sref = (ref[:, 4] * ref[:, 5])
        margin = (sref[0] - sref[1]).item() if ref.shape[0] > 1 else 1.0
        iou = orc.box_iou_np(dets[:1, :4].numpy(), ref[:1, :4].numpy())[0, 0]
        ious.append(float(iou))
        eps_all.append(eps)
        flip = iou < 0.5
        conditioned = margin > 2 * eps
        well += conditioned
        flips += flip
        hard_flips += flip and conditioned
    REPORT["sot"] = dict(frames=N_FRAMES - 1, top1_flips=int(flips), well_conditioned_frames=int(well), flips_among_well_conditioned=int(hard_flips),
                         mean_top1_iou=float(np.mean(ious)), max_score_err=float(max(eps_all)))
    print("SOT flip report:", REPORT["sot"])
    _save()
    assert hard_flips == 0, REPORT["sot"]


def _mot_models():
    import unicorn_oracle as orc
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.weights import make_state_dict
    name = "unicorn_track_tiny"
    sd = make_state_dict(name, 0)
    return name, sd, orc.CONFIGS[name], UnicornEngine(sd, name)


def test_mot_ids_from_engine_embeddings_match_oracle_embeddings():
    """The association chain that the embeddings drive — backbone -> deformable interaction with the previous frame -> embedding
    upsample -> sampling at the box centres -> bi-softmax -> QuasiDenseEmbedTracker ids (mot_evaluator.py:1014-1045) — with the
    SAME boxes on both sides (the moving objects of the synthetic video plus two static clutter boxes, fixed scores), so that the
    only difference is bf16 engine embeddings vs fp32 oracle embeddings.  Three trackers run: the product tracker and the oracle
    class on the ENGINE embeddings (must agree bit for bit on every frame: same inputs), and the oracle class on the ORACLE
    embeddings.  The last two are compared margin aware: while their states agree, a frame is well conditioned when every
    detection row's decision (lead of the best memo entry, distance from the match thresholds) is further from flipping than twice
    the largest bi-softmax score difference between the two sides; on such frames the ids must match bit for bit, and the first
    mismatch — after which the states differ and ids are no longer comparable (new tracks are numbered consecutively) — may only
    happen on an ill-conditioned frame."""
    import tracker_oracle as to
    import unicorn_oracle as orc
    from unicorn_b200 import ops
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.tracker import QuasiDenseEmbedTracker
    name, sd, cfg, eng = _mot_models()
    n_obj = 5
    frames, boxes = make_video(N_FRAMES, 320, 320, seed=11, n_obj=n_obj)
    clutter = torch.tensor([[8.0, 250.0, 60.0, 310.0], [250.0, 10.0, 310.0, 70.0]])
    scores = torch.tensor([0.95, 0.9, 0.85, 0.82, 0.6, 0.3, 0.2])  # > init 0.8: tracks start; 0.6: matched only; < 0.5: backdrops
    trk_e, trk_oe, trk_o = QuasiDenseEmbedTracker(), to.QDTrackerOracle(), to.QDTrackerOracle()
    prev_e = prev_o = None
    img_dev = torch.empty(1, 3, 320, 320, device="cuda")
    feats_dev = torch.zeros(16, 128, device="cuda")
    rows, sim_err, compared, well, first_mismatch, worst = 0, 0.0, 0, 0, None, None
    ones = torch.ones(scores.numel())
    for t in range(N_FRAMES):
        bx = torch.cat([torch.cat([boxes[t], clutter]), scores[:, None]], 1)
        # engine side
        img_dev.copy_(frames[t:t + 1])
        eng.begin_frame()
        _, seq = eng.backbone(img_dev, tag="m%d" % (t & 1))
        cur = seq["feat"].clone()
        _, f_cur = eng.interaction(prev_e if prev_e is not None else cur, cur)
        emb = eng.upsample(f_cur, "m.emb")
        prev_e = cur
        fe = ops.sample_embed(emb, bx[:, :4].cuda().contiguous(), bx.shape[0], 8.0, out=feats_dev)[:bx.shape[0]].cpu()
        # oracle side
        with torch.no_grad():
            _, oseq = orc.forward_backbone(frames[t:t + 1], sd, cfg)
            _, of_cur = orc.deform_interaction(prev_o if prev_o is not None else oseq, oseq, sd)
            fo = to.sample_embeddings(orc.upsample_embed(of_cur, sd), bx[:, :4], (320, 320))
            prev_o = oseq
        sim_err = max(sim_err, ((fe - fo).abs().max() / fo.abs().max()).item())
        if first_mismatch is None:
            s_o, margin = trk_o.decision_margin(bx.clone(), ones, fo)
            s_e, _ = trk_oe.decision_margin(bx.clone(), ones, fe)
            eps = float((s_o - s_e).abs().max()) if s_o is not None else 0.0
        be, _, ie = trk_e.match(bx.clone(), ones, fe, t + 1)
        boe, _, ioe = trk_oe.match(bx.clone(), ones, fe, t + 1)
        bo, _, io = trk_o.match(bx.clone(), ones, fo, t + 1)
        assert torch.equal(be, boe) and torch.equal(ie, ioe), (t, ie, ioe)  # product tracker == oracle class on the same inputs
        assert torch.equal(be, bo)
        rows += ie.numel()
        if first_mismatch is None:
            compared += 1
            conditioned = margin > 2 * eps
            well += conditioned
            if not torch.equal(ioe, io):
                first_mismatch = dict(frame=t, margin=margin, score_err=eps, well_conditioned=bool(conditioned))
            elif eps > 0 and (worst is None or margin / eps < worst):
                worst = margin / eps
    REPORT["mot_same_boxes"] = dict(frames=N_FRAMES, rows=rows, frames_compared=compared, well_conditioned_frames=int(well),
                                    first_mismatch=first_mismatch, smallest_margin_over_score_err=worst,
                                    tracks=int(trk_e.num_tracklets), oracle_tracks=int(trk_o.num_tracklets), max_embedding_rel_err=sim_err)
    print("MOT ids, engine vs oracle embeddings on identical boxes:", REPORT["mot_same_boxes"])
    _save()
    assert first_mismatch is None or not first_mismatch["well_conditioned"], REPORT["mot_same_boxes"]
    assert compared >= 8 and sim_err < 0.03, REPORT["mot_same_boxes"]


def test_mot_end_to_end_flip_report():
    """Raw end-to-end statistic (each side on ITS OWN detections): reported, loosely bounded.  With seeded random weights the detector
    fires on noise (scores 0.02-0.07, a different box set every frame: ~65 short-lived ids in 32 frames on BOTH sides), so id
    continuity is ill conditioned by construction; the well-conditioned halves are asserted exactly elsewhere (detections:
    tests/test_whole_gpu.py, association on identical boxes: the test above, tracker on identical detections: tests/test_tracker_gpu.py)."""
    import tracker_oracle as to
    import unicorn_oracle as orc
    from unicorn_b200.mot import UnicornMOTTracker
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.tracker import QuasiDenseEmbedTracker
    name, sd, cfg, eng = _mot_models()
    frames, _ = make_video(N_FRAMES, 320, 320, seed=5, n_obj=3)
    CONF, NMS, THR = 0.01, 0.7, 0.03
    kw = dict(init_score_thr=0.04, obj_score_thr=0.035)  # the reference's 0.8 / 0.5 scaled to the score range of seeded random weights
    trk = UnicornMOTTracker(eng, (320, 320), conf=CONF, nms=NMS, score_thr=THR, tracker=QuasiDenseEmbedTracker(**kw))
    otrk = to.QDTrackerOracle(**kw)
    prev, id_map, paired, flips, n_e, n_o = None, {}, 0, 0, 0, 0
    for t in range(N_FRAMES):
        img = frames[t:t + 1]
        eb, eid = trk.step_tensor(img)
        with torch.no_grad():
            head, seq = orc.whole_forward(img, sd, cfg)
            d = orc.postprocess(head, cfg["num_classes"], CONF, NMS)[0]
            ob, oid = torch.zeros(0, 5), torch.zeros(0, dtype=torch.long)
            if d is not None:
                sc = d[:, 4] * d[:, 5]
                keep = sc > THR
                bx = torch.cat([d[keep, :4], sc[keep, None]], 1)
                pre = prev if prev is not None else seq
                _, f_cur = orc.deform_interaction(pre, seq, sd)
                emb = orc.upsample_embed(f_cur, sd)
                prev = seq
                if bx.size(0):
                    fe = to.sample_embeddings(emb, bx[:, :4], (320, 320))
                    b2, _, i2 = otrk.match(bx, torch.ones(bx.size(0)), fe, t + 1)
                    ob, oid = b2[i2 > -1], i2[i2 > -1]
        n_e += eb.shape[0]
        n_o += ob.shape[0]
        if eb.shape[0] == 0 or ob.shape[0] == 0:
            continue
        iou = orc.box_iou_np(eb[:, :4].numpy(), ob[:, :4].numpy())
        for i in range(eb.shape[0]):
            j = int(iou[i].argmax())
            if iou[i, j] < 0.7:
                continue
            paired += 1
            e_id, o_id = int(eid[i]), int(oid[j])
            if e_id not in id_map:
                id_map[e_id] = o_id
            elif id_map[e_id] != o_id:
                flips += 1
                id_map[e_id] = o_id
    REPORT["mot"] = dict(frames=N_FRAMES, engine_track_rows=n_e, oracle_track_rows=n_o, paired_track_frames=paired, id_flips=flips,
                         distinct_engine_ids=len(id_map))
    print("MOT id flip report:", REPORT["mot"])
    _save()
    assert paired > 0.7 * min(n_e, n_o), REPORT["mot"]            # the two sides track the same boxes ...
    assert abs(n_e - n_o) <= max(3, 0.15 * n_o), REPORT["mot"]    # ... and the same number of them

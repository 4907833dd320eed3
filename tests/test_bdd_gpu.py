"""The BDD100K test protocol on the H100 (UnicornBDDMOTBatch / UnicornBDDMOTSBatch) against the unmodified qdtrack loop
(tests/golden/bdd_tiny_320.npz): the host half bit for bit on the golden's rows and embeddings, the whole driver at n_seq = 1 on the
golden's frames, the first-frame rule of QDEmbedding, n_seq = 2 and 4 against n_seq = 1, and a *_mask checkpoint in the plain
config."""
import json
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_bdd import frames, golden_bbox_result, golden_masks, split, tracked  # noqa: E402

SIZE = (320, 320)


@pytest.fixture(scope="module")
def golden():
    from test_bdd import load_bdd_golden
    return load_bdd_golden()


def tracker(g, p):
    from unicorn_b200.tracker import QuasiDenseEmbedTracker
    return QuasiDenseEmbedTracker(**json.loads(str(g[p + "tracker_cfg"])), device="cuda")


def video(g, seed=None, n=None, orig=None):
    """Letterboxed uint8 frames [n, 320, 320, 3] of make_video at the original size, quantised as the golden's are."""
    from unicorn_b200.synthetic import make_video
    oh, ow = orig or (int(v) for v in g["orig"])
    f, _ = make_video(n or int(g["n_frames"]), oh, ow, seed=int(g["seed_video"]) if seed is None else seed, n_obj=int(g["n_obj"]))
    u8 = f.round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1)
    out = torch.full((u8.shape[0], *SIZE, 3), 114, dtype=torch.uint8)
    out[:, :oh, :ow] = u8
    return out.cuda()


def same(a, b):
    """Deep equality of result dicts: keys and their order, array dtypes, shapes and values, bytes."""
    if isinstance(a, dict):
        return isinstance(b, dict) and list(a) == list(b) and all(type(k) is type(j) for k, j in zip(a, b)) and all(same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return type(a) is type(b) and len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    if isinstance(a, (np.ndarray, np.generic)):
        return type(a) is type(b) and a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b)
    return a == b


# ------------------------------------------------------------------------------------------------ host half
def test_host_half_on_the_golden_rows_is_bit_exact(golden):
    from unicorn_b200.bdd import bdd_mot_result, bdd_mots_result
    from unicorn_b200.results import rle_decode, rle_encode
    g = golden
    h, w = (int(v) for v in g["orig"])
    for p in ("mot_", "mots_"):
        t = tracker(g, p)
        feats = split(g[p + "feats"], g[p + "rows_n"])
        masks = golden_masks(g) if p == "mots_" else None
        starts = np.concatenate([[0], np.cumsum(g[p + "rows_n"])])
        tr = split(np.arange(len(g["mots_tr_id"])), g["mots_tr_n"])
        track_rows = split(g["mot_track"], g["mot_track_cls"].sum(1))
        for f, ((rows, ids, labels), boxes) in enumerate(zip(frames(g, p), tracked(g, p))):
            d, e = torch.from_numpy(rows), torch.from_numpy(feats[f])
            if p == "mot_":
                r = bdd_mot_result(t, d, e, 1.0, f, 8)
                want = split(track_rows[f], g["mot_track_cls"][f])
                dt = np.float64 if g["mot_track_f64"][f] else np.float32
                assert all(a.dtype == dt and np.array_equal(a, b.astype(dt)) for a, b in zip(r["track_results"], want)), f
                assert same(r["bbox_results"], golden_bbox_result(g, p, f))
                continue
            fm = masks[starts[f]:starts[f + 1]]
            rles = [rle_encode(m) for m in fm]
            r = bdd_mots_result(t, d, e, 1.0, f, rles, h, w, 8)
            assert same(r["bbox_result"], golden_bbox_result(g, p, f))
            assert list(r["track_result"]) == g["mots_tr_id"][tr[f]].tolist(), f
            for j, v in zip(tr[f], r["track_result"].values()):
                assert np.array_equal(v["bbox"], g["mots_tr_bbox"][j]) and v["label"] == g["mots_tr_label"][j]
                assert np.array_equal(rle_decode(v["segm"]["counts"].decode(), h, w), fm[g["mots_tr_row"][j]])
            per = [[rle_decode(s["counts"].decode(), h, w) for s in c] for c in r["segm_result"]]
            for c in range(8):  # class-wise, in NMS order
                assert len(per[c]) == int((rows[:, 6] == c).sum())
                for m, n in zip(per[c], np.flatnonzero(rows[:, 6] == c)):
                    assert np.array_equal(m, fm[n])


# ------------------------------------------------------------------------------------------------ end to end
@pytest.fixture(scope="module")
def engines():
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.weights import make_state_dict
    return {m: UnicornEngine(make_state_dict(n, 0), n) for m, n in ((False, "unicorn_track_tiny"), (True, "unicorn_track_tiny_mask"))}


def driver(engines, mots, g, n_seq=1, use_graph=True, chunk=100):
    from unicorn_b200.bdd import UnicornBDDMOTBatch, UnicornBDDMOTSBatch
    if mots:
        return UnicornBDDMOTSBatch(engines[mots], SIZE, n_seq, conf=float(g["conf"]), nms=float(g["nms"]), chunk=chunk, use_graph=use_graph)
    return UnicornBDDMOTBatch(engines[mots], SIZE, n_seq, conf=float(g["conf"]), nms=float(g["nms"]), use_graph=use_graph)


@pytest.mark.parametrize("mots", [False, True])
def test_end_to_end_on_the_golden_frames(engines, golden, mots):
    """Rows and masks against the unmodified loop, ids and labels of every frame against the reference tracker (oracle/tracker_oracle.py,
    pinned to it by tests/test_tracker_oracle.py) given the rows and embeddings the engine read back.

    The ids are not compared with the golden's: without a score filter every row enters the bisoftmax, and the seeded weights' candidate
    scores lie closer to the conf threshold, to each other's class and to the NMS threshold than the engine's bf16 error (the golden's
    recorded margins, DESIGN.md section 4.13), so the engine's row set differs from the reference's and with it the match
    confidences.  The host half on the golden's own rows is pinned bit for bit above."""
    import tracker_oracle as to
    import unicorn_oracle as orc
    from test_whole_gpu import check_dets
    from unicorn_b200.results import rle_decode, track2result
    g, p = golden, "mots_" if mots else "mot_"
    h, w = (int(v) for v in g["orig"])
    trk = driver(engines, mots, g)
    trk.start(0, tracker(g, p))
    cfg = json.loads(str(g[p + "tracker_cfg"]))
    cfg.pop("match_metric")
    oracle = to.QDTrackerOracle(**cfg)
    frs = video(g)
    masks = golden_masks(g) if mots else None
    near = g["mots_near_thr"] if mots else None
    starts = np.concatenate([[0], np.cumsum(g[p + "rows_n"])])
    ious, seen, persisted = [], set(), 0
    print(p, "detection-side decision margins of the golden:", str(g[p + "margins"]))
    for f, (rows, _, _) in enumerate(frames(g, p)):
        r = trk.step_tensor(frs[f:f + 1], [(h, w)])[0]
        d, e = trk.last_dets[0], trk.last_feats[0]
        check_dets(d, rows, orc)
        assert d.shape[0] > 0, f
        det = torch.cat([d[:, :4], d[:, 4:5] * d[:, 5:6]], 1)
        ob, ol, oid = oracle.match(det, d[:, 6].clone(), e, f)
        want = [(int(t), int(lab)) for t, lab in zip(oid, ol) if t > -1]
        persisted += sum(t in seen for t, _ in want)
        seen |= {t for t, _ in want}
        if not mots:
            assert same(r["track_results"], track2result(ob, ol, oid, 8)), f
            continue
        assert [(int(k), int(v["label"])) for k, v in r["track_result"].items()] == want, f
        valid = oid > -1
        assert all(np.array_equal(v["bbox"], b) for v, b in zip(r["track_result"].values(), ob[valid].numpy())), f
        rles = trk.last_rles[0]
        segm = [s["counts"].decode() for c in r["segm_result"] for s in c]
        assert sorted(segm) == sorted(rles)
        iou = orc.box_iou_np(d[:, :4].numpy(), rows[:, :4])
        iou[d[:, 6].numpy()[:, None] != rows[None, :, 6]] = 0.0
        for n in range(d.shape[0]):  # rows paired with the reference's by class and box; well-conditioned masks only
            j = int(iou[n].argmax())
            if iou[n, j] > 0.9 and near[starts[f] + j] < 0.05:
                a, b = rle_decode(rles[n], h, w), masks[starts[f] + j]
                union = (a | b).sum()
                ious.append(1.0 if union == 0 else (a & b).sum() / union)
    assert persisted >= 2, "the comparison must cover tracks that persist across frames"
    if mots:
        # seeded weights give some rows flat masks, where the engine's bf16 controller outputs move large areas across the threshold;
        # the rule of tests/test_inst_gpu.py: every well-conditioned row to IoU 0.95, and they are at least half of the golden's rows
        print("mask IoU of the well-conditioned rows: worst", min(ious), "of", len(ious))
        assert min(ious) >= 0.95 and len(ious) >= 0.5 * len(near), (min(ious), len(ious), len(near))


def test_segm_strings_are_inst_encode_of_the_engine_maps(engines, golden):
    """The tracked and per-class strings are those of one dynamic_masks_rows + uc_inst_encode_batched pass over the frame's rows."""
    from unicorn_b200 import ops, post_ops
    from unicorn_b200.frames import anchor_count
    from unicorn_b200.mots import MaskEncoder
    g = golden
    h, w = (int(v) for v in g["orig"])
    trk = driver(engines, True, g, use_graph=False)
    trk.start(0, tracker(g, "mots_"))
    frs = video(g, n=1)
    trk.step_tensor(frs[:1], [(h, w)])
    e = engines[True]
    ws = ops.PostWorkspace(anchor_count(*SIZE), "cuda", 1)
    e.begin_frame()
    fpn, _ = e.backbone(frs[:1], tag="bddtest")
    out = e.head(fpn, None, "mot", with_masks=True)
    ops.postprocess_device(out[0], 8, float(g["conf"]), float(g["nms"]), ws)
    mf, um = e.mask_branch(fpn)
    dyn = list(e.dyn_levels)
    n = int(ws.count[0])
    maps = torch.empty(1, n, 160, 160, device="cuda")
    post_ops.dynamic_masks_rows(mf, um, dyn, [(t.shape[1], t.shape[2]) for t in dyn], ws.anchors.view(1, -1), ws.count,
                                torch.zeros(1, dtype=torch.int32, device="cuda"), n, 4, maps, torch.empty(n * 40 * 40, device="cuda"))
    enc = MaskEncoder(n, "cuda", 1 << 20)
    enc.reserve(h, w)
    run = lambda: post_ops.inst_encode(maps, ws.count, 0, 2, 0.3, [1.0], [h], [w], enc.ws, enc.d_emit, enc.d_chars, enc.d_offsets)  # noqa: E731
    enc.enqueue(n, run)
    assert enc.strings(n, run) == trk.last_rles[0]


# ------------------------------------------------------------------------------------------------ first-frame rule
def test_first_step_rule(engines):
    from unicorn_b200.mot import QDEmbedding
    e = engines[False]
    torch.manual_seed(0)
    feats = [torch.randn(2, 20, 20, e.inc[1], device="cuda").bfloat16() for _ in range(3)]
    dets = torch.zeros(2, 2100, 7, device="cuda")
    zero = torch.zeros(2, dtype=torch.int32, device="cuda")
    for first_step in (True, False):
        qd = QDEmbedding(e, *SIZE, 16, "bddtest.emb", batch=2, first_step=first_step)
        e.begin_frame()
        qd(e, feats[0], dets, zero)  # frame 0 without detections
        torch.cuda.synchronize()
        if first_step:
            assert qd.has_prev.tolist() == [1, 1] and torch.equal(qd.prev_feat, feats[0])
        else:
            assert qd.has_prev.tolist() == [0, 0]
        e.begin_frame()
        qd(e, feats[1], dets, zero)  # a later empty step leaves pre_dict alone under the new rule
        torch.cuda.synchronize()
        if first_step:
            assert torch.equal(qd.prev_feat, feats[0])
        else:
            assert qd.has_prev.tolist() == [0, 0]
            e.begin_frame()
            qd(e, feats[2], dets, torch.tensor([1, 0], dtype=torch.int32, device="cuda"))  # today's rule: the first step with detections
            torch.cuda.synchronize()
            assert qd.has_prev.tolist() == [1, 0] and torch.equal(qd.prev_feat[0], feats[2][0])


# ------------------------------------------------------------------------------------------------ batch equality
@pytest.mark.parametrize("mots", [False, True])
@pytest.mark.parametrize("use_graph", [False, True])
def test_batch_equals_one_sequence(engines, golden, mots, use_graph):
    g, p = golden, "mots_" if mots else "mot_"
    n_frames = 5
    origs = [(288, 320), (240, 320), (320, 256), (288, 320)] if mots else [(288, 320)] * 4
    vids = [video(g, seed=10 + s, n=n_frames, orig=origs[s]) for s in range(4)]
    want = []
    for s in range(4):
        one = driver(engines, mots, g, 1, use_graph)
        one.start(0, tracker(g, p))
        want.append([one.step_tensor(vids[s][t:t + 1], [origs[s]])[0] for t in range(n_frames)])
    for n_seq in (2, 4):
        b = driver(engines, mots, g, n_seq, use_graph, chunk=4)  # several chunks per step
        got = [[] for _ in range(n_seq)]
        steps = n_frames + n_seq - 1  # sequence s starts at step s

        def collect():
            for s, r in enumerate(b.collect()):
                if r is not None:
                    got[s].append(r)
        for t in range(steps):
            if t < n_seq:
                b.start(t, tracker(g, p))
            frs = torch.stack([vids[s][min(max(t - s, 0), n_frames - 1)] for s in range(n_seq)])
            b.submit(frs, origs[:n_seq], [0 <= t - s < n_frames for s in range(n_seq)])
            if t > 0:
                collect()  # submit(t) precedes collect(t - 1)
        collect()
        for s in range(n_seq):
            assert len(got[s]) == n_frames and all(same(a, c) for a, c in zip(got[s], want[s])), (n_seq, s)


# ------------------------------------------------------------------------------------------------ checkpoint
def test_mask_checkpoint_serves_the_plain_config(golden):
    from unicorn_b200.bdd import UnicornBDDMOTBatch
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.weights import load_checkpoint, make_state_dict
    g = golden
    sd = load_checkpoint({"model": make_state_dict("unicorn_track_tiny_mask", 0)}, "unicorn_track_tiny", strict=False)
    trk = UnicornBDDMOTBatch(UnicornEngine(sd, "unicorn_track_tiny"), SIZE, 1, conf=float(g["conf"]), nms=float(g["nms"]))
    trk.start(0, tracker(g, "mot_"))
    rows, ids, labels = frames(g, "mot_")[0]
    r = trk.step_tensor(video(g, n=1), [tuple(int(v) for v in g["orig"])])[0]
    assert set(r) == {"bbox_results", "track_results"} and abs(trk.last_dets[0].shape[0] - rows.shape[0]) <= 5

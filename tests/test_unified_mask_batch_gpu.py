"""VOS objects and MOTS instances of several videos in one batched step: uc_vos_aggregate_batched against uc_vos_aggregate on each
video alone, head_shared(with_masks=True, src_of=...) over the pyramids of several images against head(..., with_masks=True) per
image, and UnicornUnifiedMaskBatch against one UnicornUnifiedMaskTracker per video, bit for bit on every step (object rows, counts and
masks, label maps, soft masks, MOTS ids / RLE strings / NMS rows / embeddings), under a schedule of objects added with and without an
init_mask, one removed and its slot reused by another video, a video idle for three steps, a video started mid-run and a video
restarted with a new original size."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_unified_mask_gpu import MOTS_KW, Video, label_map, qd_tracker, same, same_vos, snap  # noqa: E402

pytestmark = pytest.mark.gpu

TINY = (320, 320)
FULL = (800, 1280)
STEPS = 14
N_SEQ = 3
START = {0: 0, 1: 0, 2: 5}  # video -> step it is started on
IDLE = {1: {4, 5, 6}}  # video -> steps it sits out
RESTART = (11, 0)  # (step before whose submit the video is restarted, video)
# (video, step the objects are added before, {object id: object of make_video}, with an init_mask).  Video 1's object 2 is added while
# the video is idle: its reference is the video's next active frame (step 7).  Video 2's object 4 takes the slot video 0's object 2
# frees.  Object ids are per video: id 1 is in videos 0 and 1.  Video 0 is restarted on step 11 with a new original size.
ADD = [(0, 0, {1: 0, 2: 1}, False), (1, 1, {1: 0}, False), (0, 3, {3: 2}, True), (1, 5, {2: 1}, False), (2, 6, {5: 0}, True),
       (2, 9, {4: 2}, False), (0, 11, {7: 1}, False), (0, 12, {1: 0}, True)]
REMOVE = [(0, 8, 2)]  # (video, step the object is removed before, object id)
MAX_OBJECTS, MAX_GROUPS = 6, 6

_ENGINES = {}


def engine(name):
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.weights import make_state_dict
    if name not in _ENGINES:
        _ENGINES.clear()  # one engine alive at a time
        _ENGINES[name] = UnicornEngine(make_state_dict(name, 0), name)
    return _ENGINES[name]


def active_at(i, t):
    return START[i] <= t and t not in IDLE.get(i, ())


def make_videos(size, origs, n):
    """The videos of the schedule: one per video slot, plus the one video 0 is restarted on (last)."""
    return [Video(size, o, n, seed=50 + i) for i, o in enumerate(origs)]


def video_at(vids, i, t):
    return vids[-1] if i == RESTART[1] and t >= RESTART[0] else vids[i]


def adds_at(vids, i, t):
    for v, t0, objs, with_mask in ADD:
        if v == i and t0 == t:
            vid = video_at(vids, i, t)
            boxes = {oid: vid.boxes[t, o] for oid, o in objs.items()}
            yield boxes, (vid.init_mask(t, objs) if with_mask else None)


# ------------------------------------------------------------------------------------------------ kernel
def _aggregate_case(g, Hin, Win, orig, r, n_obj, kinds, ids):
    H0, W0 = orig
    masks, init = [], torch.zeros(H0, W0, dtype=torch.uint8, device="cuda")
    n_mask = 0
    for k, kind in enumerate(kinds):
        if kind == "mask":  # quantised soft values: equal values everywhere, so the argmax tie-break decides
            masks.append((torch.randint(0, 5, (1, Hin, Win), device="cuda", generator=g).float() / 4).contiguous())
            n_mask += 1
        elif kind == "empty":
            masks.append(torch.zeros(1, Hin, Win, device="cuda"))
            n_mask += 1
    # objects after the listed masks take their pixels of the init label map
    for k in range(n_mask, n_obj):
        y0, x0 = (k * 7) % (H0 // 2), (k * 13) % (W0 // 2)
        init[y0:y0 + H0 // 3, x0:x0 + W0 // 3] = ids[k]
    return masks, (init if n_mask < n_obj else None)


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("with_soft", [True, False])
def test_vos_aggregate_batched_matches_one_video_calls(B, with_soft):
    from unicorn_b200 import ops, shared_ops
    g = torch.Generator(device="cuda").manual_seed(7 + B)
    Hin, Win = 320, 320
    # (original size, r): exact covers next to ones whose floor(Hin / r) leaves an uncovered corner (hm < H or wm < W)
    shapes = [((403, 403), 0.8), ((240, 400), 0.5), ((131, 97), 2.45)][:B]
    assert int(Hin / shapes[0][1]) < shapes[0][0][0]  # video 0's bottom rows are not covered by the resize
    objs = [  # per video: (kinds, ids) with ids out of order; the objects after the masks come from the init label map
        (["mask", "empty", "mask", "init", "init"], [9, 3, 200, 1, 255]),
        (["mask"] * 8 + ["empty"] * 4 + ["init"] * 4, [16 - k for k in range(16)]),
        (["init"], [77]),
    ]
    videos, singles = [], []
    for b in range(B):
        orig, r = shapes[b]
        kinds, ids = objs[b]
        masks, init = _aggregate_case(g, Hin, Win, orig, r, len(ids), kinds, ids)
        if b == 0:
            masks[2].copy_(masks[0])  # two objects with equal soft values everywhere
        seg = torch.full(orig, 99, dtype=torch.uint8, device="cuda")
        soft = torch.full((len(ids),) + orig, -1.0, device="cuda") if with_soft else None
        videos.append((masks, init, ids, r, soft, seg))
        seg1 = seg.clone()
        soft1 = torch.full((len(ids),) + orig, -1.0, device="cuda")
        ops.vos_aggregate(masks, init, ids, Hin, Win, r, soft1, seg1)
        singles.append((seg1, soft1))
    shared_ops.vos_aggregate_batched(videos, Hin, Win)
    torch.cuda.synchronize()
    for b, ((masks, init, ids, r, soft, seg), (seg1, soft1)) in enumerate(zip(videos, singles)):
        same(seg, seg1, f"video {b} segmentation")
        if with_soft:
            same(soft, soft1, f"video {b} soft")
        assert seg.max() > 0, f"video {b}: a vacuous label map"


# ------------------------------------------------------------------------------------------------ engine
def _head_shared_case(e, mots, src, seed):
    from unicorn_b200.synthetic import make_video
    frames = torch.cat([make_video(1, *TINY, seed=40 + i, n_obj=3)[0] for i in range(N_SEQ)]).cuda()
    g = torch.Generator(device="cuda").manual_seed(seed)
    e.begin_frame()
    fpn, _ = e.backbone(frames)
    K = len(src)
    priors = [torch.rand(K, 1, f.shape[1], f.shape[2], device="cuda", generator=g) for f in fpn]
    table = torch.tensor(src, dtype=torch.int32, device="cuda")
    got_mot, got_sot = e.head_shared(fpn, priors, mot=mots, with_masks=True, src_of=table)
    got_mot = got_mot.clone() if mots else None
    got_sot = got_sot.clone()
    dyn = [t.clone() for t in e.dyn_levels]
    n_mot = N_SEQ if mots else 0
    assert all(t.shape[0] == n_mot + K and t.shape[-1] == 176 for t in dyn)
    if mots:
        for i in range(N_SEQ):
            e.begin_frame()
            same(got_mot[i:i + 1], e.head([f[i:i + 1] for f in fpn], None, "mot", with_masks=True), f"mot image {i}")
            for lvl in range(3):
                same(dyn[lvl][i:i + 1], e.dyn_levels[lvl], f"mot image {i} controllers {lvl}")
    for k, s in enumerate(src):
        e.begin_frame()
        same(got_sot[k:k + 1], e.head([f[s:s + 1] for f in fpn], [p[k] for p in priors], "sot", with_masks=True), f"object image {k} (source {s})")
        for lvl in range(3):
            same(dyn[lvl][n_mot + k:n_mot + k + 1], e.dyn_levels[lvl], f"object image {k} controllers {lvl}")


@pytest.mark.parametrize("mots", [True, False])
def test_head_shared_with_masks_and_src_of_matches_head_per_image(mots):
    _head_shared_case(engine("unicorn_track_tiny_mask"), mots, [2, 0, 2, 1], 4)


def test_head_shared_with_masks_and_src_of_one_class_mot_head():
    e = engine("unicorn_track_large_mot_challenge_mask")
    assert e.ncls == 1
    _head_shared_case(e, True, [1, 1, 0], 5)


# ------------------------------------------------------------------------------------------------ driver
def references(e, size, vids, n, mots):
    """One UnicornUnifiedMaskTracker per video (a new one for the restarted video), stepped on the video's active steps with the
    schedule's adds and removes: {(video, step): (vos snap, mots tuple, NMS rows, embeddings)}."""
    from unicorn_b200.unified import UnicornUnifiedMaskTracker
    out = {}
    for i in range(N_SEQ):
        trk = None
        for t in range(START[i], n):
            vid = video_at(vids, i, t)
            if trk is None or (i == RESTART[1] and t == RESTART[0]):
                trk = UnicornUnifiedMaskTracker(e, size, vid.orig, MAX_OBJECTS, MAX_GROUPS, mots=mots, tracker=qd_tracker() if mots else None,
                                                **MOTS_KW)
            for boxes, mask in adds_at(vids, i, t):
                trk.add_objects(boxes, init_mask=mask)
            for v, t1, oid in REMOVE:
                if v == i and t1 == t:
                    trk.remove_object(oid)
            if not active_at(i, t):
                continue
            res = trk.step_tensor(vid.frames[t:t + 1])
            counts = {oid: int(row[7]) for oid, row in trk.last_rows.items()}
            out[i, t] = (snap(res["vos"], counts), res["mots"], trk.last_dets, trk.last_feats)
    return out


def run_batch(e, size, vids, n, mots, use_graph=True, pipelined=False):
    """UnicornUnifiedMaskBatch over the videos with the schedule: per step (the results of each video, the parity graphs)."""
    from unicorn_b200.unified import UnicornUnifiedMaskBatch
    b = UnicornUnifiedMaskBatch(e, size, N_SEQ, MAX_OBJECTS, MAX_GROUPS, mots=mots, use_graph=use_graph, **MOTS_KW)
    steps, graphs = [], []

    def schedule(t):
        for i in range(N_SEQ):
            if t == START[i] or (i == RESTART[1] and t == RESTART[0]):
                b.start(i, video_at(vids, i, t).orig, qd_tracker() if mots else None)
            for boxes, mask in adds_at(vids, i, t):
                b.add_objects(i, boxes, init_mask=mask)
            for v, t1, oid in REMOVE:
                if v == i and t1 == t:
                    b.remove_object(i, oid)

    def frames(t):
        return torch.stack([video_at(vids, i, t).frames[t] if active_at(i, t) else torch.zeros_like(vids[0].frames[0])
                            for i in range(N_SEQ)])

    def active(t):
        return [active_at(i, t) for i in range(N_SEQ)]

    def record(res):
        out = []
        for i, r in enumerate(res):
            if r is None:
                out.append(None)
                continue
            counts = {oid: int(row[7]) for oid, row in b.last_rows[i].items()}
            out.append((snap(r["vos"], counts), r["mots"], b.last_dets[i], b.last_feats[i]))
        steps.append(out)
        graphs.append(b.graphs)

    if not pipelined:
        for t in range(n):
            schedule(t)
            record(b.step_tensor(frames(t), active(t)))
    else:  # submit(t + 1) before collect(t)
        schedule(0)
        b.submit(frames(0), active(0))
        for t in range(n):
            if t + 1 < n:
                schedule(t + 1)
                b.submit(frames(t + 1), active(t + 1))
            record(b.collect())
    return b, steps, graphs


def same_step(a, b, what, mots):
    same_vos(a[0], b[0], what)
    assert a[1] == b[1], (what, a[1], b[1])
    if mots:
        same(a[2], b[2], what + " NMS rows")
        same(a[3], b[3], what + " embeddings")
    else:
        assert a[1] is None and b[1] is None


def check_against_references(e, size, origs, n, mots):
    vids = make_videos(size, origs, n)
    ref = references(e, size, vids, n, mots)
    b, got, graphs = run_batch(e, size, vids, n, mots)
    n_dets = n_enc = 0
    for t in range(n):
        for i in range(N_SEQ):
            if not active_at(i, t):
                assert got[t][i] is None, (t, i)
                continue
            same_step(got[t][i], ref[i, t], f"step {t} video {i}", mots)
            n_dets += sum(c > 0 for c in got[t][i][0]["counts"].values())
            if mots:
                n_enc += len(got[t][i][1][5])
    assert n_dets > 0, "no VOS detections: a vacuous test"
    assert not mots or n_enc > 0, "no MOTS instance was encoded: a vacuous test"
    # the first step runs eagerly, each parity slot's next step is captured; starts, adds, removes and idle steps never re-capture
    assert graphs[0] == [None, None] and graphs[1][0] is None and graphs[1][1] is not None
    assert all(g[0] is graphs[2][0] and g[1] is graphs[2][1] for g in graphs[2:]) and graphs[2][0] is not None
    return vids, got


TINY_ORIGS = [(320, 320), (240, 400), (403, 403), (400, 300)]  # the videos of slots 0..2, then video 0's restart


@pytest.mark.parametrize("mots", [True, False])
def test_unified_mask_batch_tiny_matches_one_tracker_per_video(mots):
    e = engine("unicorn_track_tiny_mask")
    vids, got = check_against_references(e, TINY, TINY_ORIGS, STEPS, mots)
    # eager equals graph, and the pipelined protocol (submit(t + 1) before collect(t)) equals the sequential one
    for use_graph in (False, True):
        _, other, _ = run_batch(e, TINY, vids, STEPS, mots, use_graph=use_graph, pipelined=True)
        for t, (a, b) in enumerate(zip(got, other)):
            for i in range(N_SEQ):
                assert (a[i] is None) == (b[i] is None), (t, i)
                if a[i] is not None:
                    same_step(a[i], b[i], f"use_graph={use_graph} pipelined step {t} video {i}", mots)
    # the schedule did what it says: video 0 lost object 2, video 2's object 4 reuses its slot, video 1's object 2 waited
    assert got[7][0][0]["ids"] == [1, 2, 3] and got[8][0][0]["ids"] == [1, 3]
    assert got[7][1][0]["ids"] == [1] and got[8][1][0]["ids"] == [1, 2]
    assert got[12][0][0]["ids"] == [7, 1] and tuple(got[12][0][0]["seg"].shape) == TINY_ORIGS[3]


def test_unified_mask_batch_large_full_size_matches_one_tracker_per_video():
    """unicorn_track_large_mask at 800x1280 from 1080x1920 frames (r = 2/3), and a 720x1280 restart."""
    check_against_references(engine("unicorn_track_large_mask"), FULL, [(1080, 1920)] * 3 + [(720, 1280)], 12, True)


def test_unified_mask_batch_r50_matches_one_tracker_per_video():
    check_against_references(engine("unicorn_track_r50_mask"), TINY, TINY_ORIGS, 13, True)


def test_free_slot_contents_do_not_change_live_objects():
    """Free object and group slots compute on whatever their buffers hold: garbage there changes no live result."""
    from unicorn_b200.unified import UnicornUnifiedMaskBatch
    e = engine("unicorn_track_tiny_mask")
    vids = make_videos(TINY, [(320, 320), (240, 400)], 5)
    runs = []
    for garbage in (False, True):
        b = UnicornUnifiedMaskBatch(e, TINY, 2, 4, 4, mots=True, **MOTS_KW)
        for i in range(2):
            b.start(i, vids[i].orig, qd_tracker())
            b.add_objects(i, {1: vids[i].boxes[0, 0]})
        frames = lambda t: torch.stack([v.frames[t] for v in vids])  # noqa: E731
        b.step_tensor(frames(0))
        if garbage:
            n = b.ref_proj[0].shape[0] // 4
            b.ref_proj[0][2 * n:].normal_()
            b.ref_proj[1][2 * n:].normal_()
            b.lbs[2:].uniform_()
            b.obj_row[2:].fill_(2 * b.R + 1)  # the free object slots read a row of a free group slot
            b.obj_seq[2:].fill_(1)
            b.group_seq[2:].fill_(1)
            for s in b._ring.slots:
                s.vos_masks[2:].fill_(0.75)
        res = []
        for t in range(1, 5):
            out = b.step_tensor(frames(t))
            res.append([(snap(o["vos"], {k: int(r[7]) for k, r in b.last_rows[i].items()}), o["mots"]) for i, o in enumerate(out)])
            assert b.vos_ws.count[2:].eq(0).all()  # the free slots' counts are zeroed on the device
        runs.append(res)
    for t, (a, c) in enumerate(zip(*runs)):
        for i in range(2):
            assert a[i][0]["ids"] == [1]
            same_vos(a[i][0], c[i][0], f"step {t + 1} video {i}")
            assert a[i][1] == c[i][1]


def test_reference_protocol_matches_one_tracker_per_video():
    """track(images, infos) letterboxes each video's frame once: its label maps, MOTS tuples and states equal those of one
    UnicornUnifiedMaskTracker.track per video (video 1 idle on step 2)."""
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.unified import UnicornUnifiedMaskBatch, UnicornUnifiedMaskTracker
    e = engine("unicorn_track_tiny_mask")
    origs = [(240, 400), (320, 256)]
    xywh = lambda b: [float(b[0]), float(b[1]), float(b[2] - b[0]), float(b[3] - b[1])]  # noqa: E731
    imgs, infos = [], []
    for i, orig in enumerate(origs):
        frames, boxes = make_video(5, *orig, seed=60 + i, n_obj=3)
        imgs.append([f.permute(1, 2, 0).flip(-1).round().clamp(0, 255).to(torch.uint8).numpy().copy() for f in frames])
        first = {"init_object_ids": ["1", "2"], "init_bbox": {"1": xywh(boxes[0, 0]), "2": xywh(boxes[0, 1])}}
        later = {"init_object_ids": ["3"], "init_bbox": {"3": xywh(boxes[3, 2])}, "init_mask": label_map(boxes[3, 2], 3, *orig).numpy()}
        infos.append({0: first, 3: later})
    idle = {(1, 2)}
    ref = {}
    for i, orig in enumerate(origs):
        trk = UnicornUnifiedMaskTracker(e, TINY, orig, 3, 2, tracker=qd_tracker(), **MOTS_KW)
        for t in range(5):
            if (i, t) in idle:
                continue
            out = trk.track(imgs[i][t], infos[i].get(t))
            ref[i, t] = (out, dict(trk.state_pre_dict))
    b = UnicornUnifiedMaskBatch(e, TINY, 2, 6, 4, **MOTS_KW)
    for i, orig in enumerate(origs):
        b.start(i, orig, qd_tracker())
    for t in range(5):
        out = b.track([None if (i, t) in idle else imgs[i][t] for i in range(2)], [infos[i].get(t) for i in range(2)])
        for i in range(2):
            if (i, t) in idle:
                assert out[i] is None
                continue
            want, states = ref[i, t]
            assert np.array_equal(out[i]["segmentation"], want["segmentation"]), (t, i)
            assert out[i]["mots"] == want["mots"], (t, i)
            assert b.state_pre_dicts[i] == states, (t, i)
    assert out[0]["segmentation"].max() > 0


def test_rejections_change_nothing():
    from unicorn_b200.unified import UnicornUnifiedMaskBatch
    e = engine("unicorn_track_tiny_mask")
    vids = make_videos(TINY, [(320, 320), (240, 400)], 2)
    b = UnicornUnifiedMaskBatch(e, TINY, 2, 6, 3, mots=False)
    b.start(0, vids[0].orig)
    b.add_objects(0, {1: vids[0].boxes[0, 0], 2: vids[0].boxes[0, 1]})
    frames = torch.stack([v.frames[0] for v in vids])

    def state():
        return ([b.objects(i) for i in range(2)], [[(list(x), m is None) for x, m in p] for p in b._pending], list(b._os), list(b._gs),
                b._ring.submitted, list(b.frame_ids), list(b.started), list(b.orig_sizes), b.image_of.tolist(), b.obj_row.tolist(),
                b.obj_seq.tolist(), b.group_seq.tolist())
    before = state()
    box = vids[0].boxes[0, 2]
    with pytest.raises(ValueError, match="duplicate"):
        b.add_objects(0, {1: box})
    with pytest.raises(ValueError, match="duplicate"):
        b.add_objects(0, {4: box, "4": box})
    with pytest.raises(ValueError, match="1..255"):
        b.add_objects(0, {0: box})
    with pytest.raises(ValueError, match="1..255"):
        b.add_objects(0, {256: box})
    with pytest.raises(ValueError, match="max_objects"):
        b.add_objects(0, {o: box for o in range(4, 9)})
    with pytest.raises(ValueError, match="4 values"):
        b.add_objects(0, {4: [0.0, 1.0, 2.0]})
    with pytest.raises(ValueError, match="init_mask"):
        b.add_objects(0, {4: box}, init_mask=torch.zeros(240, 400, dtype=torch.uint8))
    with pytest.raises(ValueError, match="init_mask"):
        b.add_objects(0, {4: box}, init_mask=torch.zeros(TINY, dtype=torch.int64))
    with pytest.raises(ValueError, match="not been started"):
        b.add_objects(1, {4: box})
    with pytest.raises(ValueError, match="unknown video"):
        b.add_objects(2, {4: box})
    with pytest.raises(ValueError, match="unknown object"):
        b.remove_object(0, 7)
    with pytest.raises(ValueError, match="orig_size"):
        b.start(1, (0, 400))
    with pytest.raises(ValueError, match="unknown video"):
        b.start(-1, (240, 400))
    with pytest.raises(ValueError, match="frame must be"):
        b.submit(frames[:1])
    with pytest.raises(ValueError, match="not been started"):
        b.submit(frames, [True, True])
    with pytest.raises(ValueError, match="active has"):
        b.submit(frames, [True])
    with pytest.raises(ValueError, match="size"):
        b.track([np.zeros((240, 400, 3), np.uint8), None])
    with pytest.raises(ValueError, match="not been started"):
        b.track([None, np.zeros((240, 400, 3), np.uint8)])
    assert state() == before
    b.add_objects(0, {3: box}, init_mask=torch.zeros(TINY, dtype=torch.uint8))
    before = state()
    with pytest.raises(ValueError, match="already has an init_mask"):
        b.add_objects(0, {4: box}, init_mask=torch.zeros(TINY, dtype=torch.uint8))
    with pytest.raises(ValueError, match="at most 16"):
        b.add_objects(0, {o: box for o in range(10, 24)})
    b.start(1, vids[1].orig)
    before = state()
    with pytest.raises(ValueError, match="max_groups"):  # one group slot is free, the two videos' requests need two
        b.track([vids[0].frames[0].numpy()[..., ::-1].copy() * 0, np.zeros((240, 400, 3), np.uint8)],
                [{"init_object_ids": [4], "init_bbox": {4: [0, 0, 8, 8]}}, {"init_object_ids": [1], "init_bbox": {1: [0, 0, 8, 8]}}])
    assert state() == before
    # the batch still runs on the state it had: step 0 is the reference of objects 1..3 of video 0, object 3 enters from its mask
    res = b.step_tensor(frames, [True, False])
    assert res[1] is None and res[0]["vos"]["ids"] == [3] and res[0]["mots"] is None and b.objects(0) == [1, 2, 3]
    # a step with no active video launches nothing and reports nothing
    assert b.step_tensor(frames, [False, False]) == [None, None]


@pytest.mark.parametrize("name", ["unicorn_track_tiny", "unicorn_det_convnext_tiny"])
def test_configs_without_the_tracking_mask_head_are_rejected(name):
    from unicorn_b200.unified import UnicornUnifiedMaskBatch
    with pytest.raises(ValueError, match="mask"):
        UnicornUnifiedMaskBatch(engine(name), TINY, 2, 1)

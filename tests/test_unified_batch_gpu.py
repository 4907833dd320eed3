"""SOT targets and MOT objects of several videos in one batched step: the gathering stem GroupNorm against uc_groupnorm_apply at B = 1,
head_shared over the pyramids of several images against head() at B = 1 per image, and UnicornUnifiedBatch against one
UnicornUnifiedTracker per video, bit for bit on every step (per-target detections and counts, MOT boxes / ids / NMS rows / embeddings
or ByteTrack tracks), under a schedule of targets added and removed, a video idle for some steps and a video started mid-run."""
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

TINY = (320, 320)
FULL = (800, 1280)
STEPS = 14
MOT_KW = dict(conf=0.01, nms=0.7, score_thr=0.02)
N_SEQ = 3
START = {0: 0, 1: 0, 2: 5}  # video -> step it is started on
IDLE = {1: {4, 5, 6}}  # video -> steps it sits out
# (video, target id, step it is added before, object of the video's make_video); target ids are per video: "a" is in videos 0 and 1.
# Video 1's "e" is added while the video is idle: its reference is the video's next active frame (step 7).  Video 2's "d" takes the
# slot video 0's "b" frees, so a slot changes video.
ADD = [(0, "a", 0, 0), (1, "a", 1, 0), (0, "b", 2, 1), (1, "e", 5, 1), (2, "c", 6, 0), (2, "d", 9, 2)]
REMOVE = [(0, "b", 8)]  # (video, target id, step it is removed before)
MAX_TARGETS = 5


def bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def same(a, b, what=""):
    assert a.shape == b.shape, (what, a.shape, b.shape)
    assert torch.equal(bits(a), bits(b)), (what, (a.float() - b.float()).abs().max().item())


_ENGINES = {}


def engine(name):
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.weights import make_state_dict
    if name not in _ENGINES:
        _ENGINES.clear()  # one engine alive at a time
        _ENGINES[name] = UnicornEngine(make_state_dict(name, 0), name)
    return _ENGINES[name]


def videos(size, n=STEPS):
    from unicorn_b200.synthetic import make_video
    return [make_video(n, *size, seed=40 + i, n_obj=6) for i in range(N_SEQ)]


def qd_tracker():
    from unicorn_b200.tracker import QuasiDenseEmbedTracker
    # seeded weights give low scores: lower the score gates so that tracklets are created (as tests/test_unified_gpu.py)
    return QuasiDenseEmbedTracker(init_score_thr=0.05, obj_score_thr=0.03)


def byte_tracker():
    from unicorn_b200.tracker import BYTETracker
    return BYTETracker(types.SimpleNamespace(track_thresh=0.05, track_buffer=30, match_thresh=0.9, mot20=False))


def new_tracker(mot):
    return {"qd": qd_tracker, "byte": byte_tracker, None: lambda: None}[mot]()


def byte_rows(tracks):
    # track ids come from one process-wide counter (STrack.next_id), so trackers stepped in another order number their tracks
    # differently: the boxes and scores of the active tracks, in the tracker's order, are compared
    return np.array([[*t.tlwh, t.score] for t in tracks], dtype=np.float64).reshape(-1, 5)


def active_at(i, t):
    return START[i] <= t and t not in IDLE.get(i, ())


# ------------------------------------------------------------------------------------------------ kernel
def _gather_case(g, n_src=3, h=12, w=20, C=256, G_=16):
    wide = torch.randn(n_src, h, w, C + 64, device="cuda", generator=g).bfloat16()
    x = wide[..., 32:32 + C]  # a channel slice: pixel stride C + 64
    x[:, 0, 0] = -300.0  # with the large weights below, SiLU of these pixels is -0.0 in the images without a prior
    xs = x.float().reshape(n_src, h * w, G_, C // G_)
    fix = 1 << 22
    st = torch.stack([(xs.sum(dim=(1, 3)) * fix).round().long(), ((xs * xs).sum(dim=(1, 3)) * fix).round().long()], -1).contiguous()
    gw = torch.randn(C, device="cuda", generator=g)
    gw[:16] = 100.0
    gb = torch.randn(C, device="cuda", generator=g)
    beta = torch.randn(C, device="cuda", generator=g)
    return x, st, gw, gb, beta


def _gather_reference(x, st, gw, gb, beta, act, n_plain, src, prior):
    from unicorn_b200 import ops
    _, h, w, C = x.shape
    refs = []
    for b, s in enumerate(src):
        ref = torch.empty(1, h, w, C, dtype=torch.bfloat16, device="cuda")
        pr = prior[b - n_plain].reshape(-1).contiguous() if b >= n_plain else None
        ops.groupnorm_apply(x[s:s + 1], st[s], gw, gb, st.shape[1], 1e-3, act, out=ref, prior=pr, beta=beta if pr is not None else None)
        refs.append(ref)
    return refs


@pytest.mark.parametrize("act", [0, 1, 3])
@pytest.mark.parametrize("src", [[2, 0, 1, 1, 2], [1, 1, 1, 0, 0], [0, 1, 2, 2, 1]])
@pytest.mark.parametrize("n_plain", [0, 2, 5])
def test_gather_stem_matches_groupnorm_apply(act, src, n_plain):
    from unicorn_b200 import shared_ops
    g = torch.Generator(device="cuda").manual_seed(1)
    x, st, gw, gb, beta = _gather_case(g)
    _, h, w, C = x.shape
    B = len(src)
    prior = torch.rand(max(B - n_plain, 1), 1, h, w, device="cuda", generator=g)
    if B - n_plain > 1:
        prior[1] = 0.0  # a zero prior plane still takes the prior path, as its own B = 1 call does
    table = torch.tensor(src, dtype=torch.int32, device="cuda")
    out = torch.full((B, h, w, C), 7.0, dtype=torch.bfloat16, device="cuda")
    pr = prior[:B - n_plain].reshape(-1) if n_plain < B else None
    shared_ops.groupnorm_apply_gather(x, st, gw, gb, st.shape[1], 1e-3, act, out, n_plain, table, prior=pr,
                                      beta=beta if pr is not None else None)
    for b, ref in enumerate(_gather_reference(x, st, gw, gb, beta, act, n_plain, src, prior)):
        same(out[b:b + 1], ref, f"image {b} (source {src[b]})")
    if act == 3 and n_plain > 0:  # the no-prior images keep their negative zeros
        assert (bits(out[:n_plain]) == -32768).any()


def test_gather_out_of_range_entry_leaves_its_image_untouched():
    from unicorn_b200 import shared_ops
    g = torch.Generator(device="cuda").manual_seed(2)
    x, st, gw, gb, beta = _gather_case(g)
    _, h, w, C = x.shape
    src = [1, 3, -1, 0, 65535]
    prior = torch.rand(3, 1, h, w, device="cuda", generator=g)
    out = torch.randn(len(src), h, w, C, device="cuda", generator=g).bfloat16()
    before = out.clone()
    shared_ops.groupnorm_apply_gather(x, st, gw, gb, st.shape[1], 1e-3, 3, out, 2, torch.tensor(src, dtype=torch.int32, device="cuda"),
                                      prior=prior.reshape(-1), beta=beta)
    refs = _gather_reference(x, st, gw, gb, beta, 3, 2, [1, 0, 0, 0, 0], prior)
    for b in (1, 2, 4):
        same(out[b], before[b], f"image {b} (out-of-range entry)")
    same(out[0:1], refs[0], "image 0")
    same(out[3:4], refs[3], "image 3")


def test_gather_graph_follows_the_table():
    from unicorn_b200 import shared_ops
    g = torch.Generator(device="cuda").manual_seed(3)
    x, st, gw, gb, beta = _gather_case(g)
    _, h, w, C = x.shape
    prior = torch.rand(3, 1, h, w, device="cuda", generator=g)
    table = torch.tensor([0, 1, 2, 0], dtype=torch.int32, device="cuda")
    out = torch.zeros(4, h, w, C, dtype=torch.bfloat16, device="cuda")
    run = lambda: shared_ops.groupnorm_apply_gather(x, st, gw, gb, st.shape[1], 1e-3, 1, out, 1, table, prior=prior.reshape(-1),  # noqa: E731
                                                    beta=beta)
    run()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        run()
    for src in ([2, 2, 0, 1], [1, 0, 1, 2]):
        table.copy_(torch.tensor(src, dtype=torch.int32))
        graph.replay()
        for b, ref in enumerate(_gather_reference(x, st, gw, gb, beta, 1, 1, src, prior)):
            same(out[b:b + 1], ref, f"table {src} image {b}")


# ------------------------------------------------------------------------------------------------ engine
def _head_shared_case(e, mot, src, seed):
    vids = videos(TINY, n=1)
    frames = torch.cat([v[0][:1] for v in vids]).cuda()
    g = torch.Generator(device="cuda").manual_seed(seed)
    e.begin_frame()
    fpn, _ = e.backbone(frames)
    K = len(src)
    priors = [torch.rand(K, 1, f.shape[1], f.shape[2], device="cuda", generator=g) for f in fpn]
    table = torch.tensor(src, dtype=torch.int32, device="cuda")
    got_mot, got_sot = e.head_shared(fpn, priors, mot=mot, src_of=table)
    got_mot = got_mot.clone() if mot else None
    got_sot = got_sot.clone()
    assert got_sot.shape[0] == K
    if mot:
        assert got_mot.shape[:1] == (N_SEQ,) and got_mot.shape[-1] == 5 + e.ncls
        for i in range(N_SEQ):
            e.begin_frame()
            same(got_mot[i:i + 1], e.head([f[i:i + 1] for f in fpn], None, "mot"), f"mot image {i}")
    for k, s in enumerate(src):
        e.begin_frame()
        same(got_sot[k:k + 1], e.head([f[s:s + 1] for f in fpn], [p[k] for p in priors], "sot"), f"sot image {k} (source {s})")


@pytest.mark.parametrize("mot", [True, False])
def test_head_shared_gather_matches_head_per_image(mot):
    _head_shared_case(engine("unicorn_track_tiny"), mot, [2, 0, 0, 1], 4)


def test_head_shared_gather_one_class_mot_head():
    """unicorn_track_large_mot_challenge: 1-class MOT heads next to 1-class SOT heads, each decoded into its own buffer."""
    e = engine("unicorn_track_large_mot_challenge")
    assert e.ncls == 1
    _head_shared_case(e, True, [1, 2], 5)


# ------------------------------------------------------------------------------------------------ driver
def references(e, size, vids, mot, kw):
    """One UnicornUnifiedTracker per video, stepped on the video's active steps with the schedule's adds and removes: {(video, step):
    (targets, mot result, NMS rows, embeddings)}."""
    from unicorn_b200.unified import UnicornUnifiedTracker
    out = {}
    for i, (frames, boxes) in enumerate(vids):
        trk = UnicornUnifiedTracker(e, size, 3, mot=mot, tracker=new_tracker(mot), mot_conf=kw["conf"], mot_nms=kw["nms"],
                                    score_thr=kw["score_thr"])
        for t in range(START[i], len(frames)):
            for v, tid, t0, obj in ADD:
                if v == i and t0 == t:
                    trk.add_target(tid, boxes[t, obj])
            for v, tid, t1 in REMOVE:
                if v == i and t1 == t:
                    trk.remove_target(tid)
            if not active_at(i, t):
                continue
            res = trk.step_tensor(frames[t:t + 1], img_info=size)
            m = byte_rows(res["mot"]) if mot == "byte" else res["mot"]
            out[i, t] = (res["targets"], m, trk.last_dets, trk.last_feats)
    return out


def run_batch(e, size, vids, mot, kw, use_graph=True, pipelined=False):
    """UnicornUnifiedBatch over the videos with the schedule: per step (results, last_dets, last_feats) and the graph after the step."""
    from unicorn_b200.unified import UnicornUnifiedBatch
    n = len(vids[0][0])
    trk = UnicornUnifiedBatch(e, size, N_SEQ, MAX_TARGETS, mot=mot, mot_conf=kw["conf"], mot_nms=kw["nms"], score_thr=kw["score_thr"],
                              use_graph=use_graph)
    frames = [torch.stack([v[0][t] for v in vids]) for t in range(n)]
    out, graphs = [], []

    def schedule(t):
        for i, t0 in START.items():
            if t0 == t:
                trk.start(i, new_tracker(mot))
        for i, tid, t0, obj in ADD:
            if t0 == t:
                trk.add_target(i, tid, vids[i][1][t, obj])
        for i, tid, t1 in REMOVE:
            if t1 == t:
                trk.remove_target(i, tid)
        return [active_at(i, t) for i in range(N_SEQ)]

    def record(res):
        for r in res:
            if r is not None and mot == "byte":
                r["mot"] = byte_rows(r["mot"])
        out.append((res, list(trk.last_dets), list(trk.last_feats)))

    if not pipelined:
        for t in range(n):
            record(trk.step_tensor(frames[t], active=schedule(t), img_infos=[size] * N_SEQ))
            graphs.append(trk.graph)
    else:  # submit(t + 1) before collect(t)
        trk.submit(frames[0], active=schedule(0))
        for t in range(n):
            if t + 1 < n:
                trk.submit(frames[t + 1], active=schedule(t + 1))
            graphs.append(trk.graph)
            record(trk.collect([size] * N_SEQ))
    assert trk._ring.submitted == trk._ring.collected == n
    return out, graphs


def same_results(a, b, mot, what):
    """Two runs' per-step results (results, last_dets, last_feats), bit for bit."""
    for t, ((ra, da, fa), (rb, db, fb)) in enumerate(zip(a, b)):
        for i in range(N_SEQ):
            assert (ra[i] is None) == (rb[i] is None), (what, t, i)
            if ra[i] is None:
                continue
            assert ra[i]["targets"].keys() == rb[i]["targets"].keys(), (what, t, i)
            for tid in ra[i]["targets"]:
                same(ra[i]["targets"][tid][0], rb[i]["targets"][tid][0], f"{what} step {t} video {i} target {tid}")
                assert ra[i]["targets"][tid][1] == rb[i]["targets"][tid][1], (what, t, i, tid)
            if mot is not None:
                same(da[i], db[i], f"{what} step {t} video {i} NMS rows")
            if mot == "qd":
                same(fa[i], fb[i], f"{what} step {t} video {i} embeddings")
                same(ra[i]["mot"][0], rb[i]["mot"][0], f"{what} step {t} video {i} boxes")
                assert torch.equal(ra[i]["mot"][1], rb[i]["mot"][1]), (what, t, i)
            elif mot == "byte":
                assert np.array_equal(ra[i]["mot"], rb[i]["mot"]), (what, t, i)


def check_against_references(e, size, mot, n=STEPS, kw=MOT_KW):
    vids = videos(size, n)
    ref = references(e, size, vids, mot, kw)
    got, graphs = run_batch(e, size, vids, mot, kw)
    n_sot = n_mot = 0
    for t, (res, dets, feats) in enumerate(got):
        for i in range(N_SEQ):
            if not active_at(i, t):
                assert res[i] is None, (t, i)
                continue
            rt, rm, rdets, rfeats = ref[i, t]
            assert res[i]["targets"].keys() == rt.keys(), (t, i, res[i]["targets"].keys(), rt.keys())
            for tid, (rd, rn) in rt.items():
                gd, gn = res[i]["targets"][tid]
                assert gn == rn, (t, i, tid, gn, rn)
                same(gd, rd, f"step {t} video {i} target {tid} dets")
                n_sot += rn
            if mot is None:
                assert res[i]["mot"] is None
                continue
            same(dets[i], rdets, f"step {t} video {i} NMS rows")
            n_mot += rdets.shape[0]
            if mot == "qd":
                same(feats[i], rfeats, f"step {t} video {i} embeddings")
                same(res[i]["mot"][0], rm[0], f"step {t} video {i} boxes")
                assert torch.equal(res[i]["mot"][1], rm[1]), (t, i, res[i]["mot"][1], rm[1])
            else:
                assert np.array_equal(res[i]["mot"], rm), (t, i, res[i]["mot"], rm)
    assert n_sot > 0, "no SOT detections: a vacuous test"
    assert mot is None or n_mot > 0, "no MOT detections: a vacuous test"
    # every target is reported on the steps the schedule says
    assert set(got[7][0][1]["targets"]) == {"a"} and set(got[8][0][1]["targets"]) == {"a", "e"}
    assert set(got[9][0][2]["targets"]) == {"c"} and set(got[10][0][2]["targets"]) == {"c", "d"}
    # first step eager, second captured; every later add, remove, start and activity change keeps that graph
    assert graphs[0] is None and graphs[1] is not None and all(g is graphs[1] for g in graphs[1:])
    return vids, got


@pytest.mark.parametrize("mot", ["qd", "byte", None])
def test_batch_tiny_matches_one_tracker_per_video(mot):
    e = engine("unicorn_track_tiny")
    vids, got = check_against_references(e, TINY, mot)
    eager, graphs = run_batch(e, TINY, vids, mot, MOT_KW, use_graph=False)
    assert all(g is None for g in graphs)
    same_results(got, eager, mot, "eager")
    for use_graph in (True, False):
        piped, _ = run_batch(e, TINY, vids, mot, MOT_KW, use_graph=use_graph, pipelined=True)
        same_results(got, piped, mot, f"pipelined (graph {use_graph})")


def test_batch_large_full_size_matches_one_tracker_per_video():
    check_against_references(engine("unicorn_track_large"), FULL, "qd", n=11)


def test_batch_r50_matches_one_tracker_per_video():
    check_against_references(engine("unicorn_track_r50"), TINY, "qd", n=11)


def test_reference_protocol_matches_one_tracker_per_video():
    """track(images, new_targets) letterboxes each video's frame once, at its own original size: its states and MOT output equal those
    of one UnicornUnifiedTracker.track per video; an idle video gets None."""
    from unicorn_b200.unified import UnicornUnifiedBatch, UnicornUnifiedTracker
    e = engine("unicorn_track_tiny")
    sizes = [(240, 400), (320, 320)]
    vids = []
    for k, (h, w) in enumerate(sizes):
        from unicorn_b200.synthetic import make_video
        frames, boxes = make_video(5, h, w, seed=50 + k, n_obj=3)
        vids.append(([f.permute(1, 2, 0).flip(-1).round().to(torch.uint8).numpy().copy() for f in frames], boxes))
    xywh = lambda b: [float(b[0]), float(b[1]), float(b[2] - b[0]), float(b[3] - b[1])]  # noqa: E731
    new = {0: {1: {"a": xywh(vids[0][1][1, 0])}}, 1: {0: {"a": xywh(vids[1][1][0, 1])}}}  # step -> {video: {tid: xywh}}
    idle = {(1, 2)}  # (video, step)
    kw = dict(mot_conf=MOT_KW["conf"], mot_nms=MOT_KW["nms"], score_thr=MOT_KW["score_thr"])
    ref = {}
    for i, (imgs, _) in enumerate(vids):
        trk = UnicornUnifiedTracker(e, TINY, 2, mot="qd", tracker=qd_tracker(), **kw)
        for t, im in enumerate(imgs):
            if (i, t) not in idle:
                ref[i, t] = trk.track(im, new_targets=new.get(t, {}).get(i))
    bt = UnicornUnifiedBatch(e, TINY, 2, 3, mot="qd", **kw)
    for i in range(2):
        bt.start(i, qd_tracker())
    for t in range(5):
        out = bt.track([None if (i, t) in idle else vids[i][0][t] for i in range(2)], new_targets=new.get(t))
        for i in range(2):
            if (i, t) in idle:
                assert out[i] is None
                continue
            assert out[i]["targets"] == ref[i, t]["targets"], (t, i)
            same(out[i]["mot"][0], ref[i, t]["mot"][0], f"step {t} video {i} boxes")
            assert torch.equal(out[i]["mot"][1], ref[i, t]["mot"][1])
    assert any(ref[i, t]["targets"] for i, t in ref)


def test_rejections_change_nothing():
    from unicorn_b200.unified import UnicornUnifiedBatch
    e = engine("unicorn_track_tiny")
    vids = videos(TINY, n=1)
    boxes = vids[0][1]
    with pytest.raises(ValueError, match="mot must be"):
        UnicornUnifiedBatch(e, TINY, 2, 2, mot="sort")
    with pytest.raises(ValueError, match=">= 1"):
        UnicornUnifiedBatch(e, TINY, 0, 2)
    byte = UnicornUnifiedBatch(e, TINY, 2, 2, mot="byte")
    with pytest.raises(ValueError, match="BYTETracker"):
        byte.start(0)
    assert byte.started == [False, False]
    trk = UnicornUnifiedBatch(e, TINY, 2, 3, mot=None)
    with pytest.raises(ValueError, match="not been started"):
        trk.add_target(0, "a", boxes[0, 0])
    trk.start(0)
    for i in (2, -1, "0", None):
        with pytest.raises(ValueError, match="unknown video"):
            trk.start(i)
        with pytest.raises(ValueError, match="unknown video"):
            trk.add_target(i, "a", boxes[0, 0])
        with pytest.raises(ValueError, match="unknown video"):
            trk.remove_target(i, "a")
    trk.add_target(0, "a", boxes[0, 0])
    with pytest.raises(ValueError, match="duplicate"):
        trk.add_target(0, "a", boxes[0, 1])
    with pytest.raises(ValueError, match="needs 4 values"):
        trk.add_target(0, "b", [0, 0, 1])
    trk.add_target(0, "b", boxes[0, 1])
    trk.start(1)
    trk.add_target(1, "a", boxes[0, 2])  # the same id in another video
    with pytest.raises(ValueError, match="exceed max_targets"):
        trk.add_target(1, "c", boxes[0, 3])
    with pytest.raises(ValueError, match="unknown target"):
        trk.remove_target(1, "b")
    frames = torch.zeros(2, 3, *TINY)
    with pytest.raises(ValueError, match="frame must be"):
        trk.submit(frames[:, :, :160])
    with pytest.raises(ValueError, match="frame must be"):
        trk.submit(frames[:1])
    with pytest.raises(ValueError, match="scales"):
        trk.submit(frames, scales=[1.0])
    with pytest.raises(ValueError, match="active has"):
        trk.submit(frames, active=[True])
    img = np.zeros((320, 320, 3), np.uint8)
    with pytest.raises(ValueError, match="frames for 2 videos"):
        trk.track([img])
    with pytest.raises(ValueError, match="RGB uint8"):
        trk.track([img[..., :2], None])
    with pytest.raises(ValueError, match="duplicate"):
        trk.track([img, None], new_targets={0: {"a": [0, 0, 10, 10]}})
    with pytest.raises(ValueError, match="exceed max_targets"):
        trk.track([img, img], new_targets={0: {"c": [0, 0, 10, 10]}})
    with pytest.raises(ValueError, match="unknown video"):
        trk.track([img, img], new_targets={2: {"c": [0, 0, 10, 10]}})
    assert trk.targets(0) == ["a", "b"] and trk.targets(1) == ["a"] and trk._ring.submitted == 0 and sorted(trk._pending) == [0, 1, 2]
    one = UnicornUnifiedBatch(e, TINY, 2, 1, mot=None)
    one.start(0)
    with pytest.raises(ValueError, match="not been started"):
        one.submit(frames, active=[True, True])
    with pytest.raises(ValueError, match="not been started"):
        one.track([img, img])
    assert one._ring.submitted == 0


def test_detector_config_is_rejected():
    from unicorn_b200.unified import UnicornUnifiedBatch
    with pytest.raises(ValueError, match="detector"):
        UnicornUnifiedBatch(engine("unicorn_det_convnext_tiny"), TINY, 2, 1)

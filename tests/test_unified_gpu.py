"""One backbone pass per frame for SOT targets and a MOT arm: the one-image stem GroupNorm (the gather with a table of zeros) against
uc_groupnorm_apply, the shared-trunk head against head() at B = 1, and UnicornUnifiedTracker (UnicornUnifiedBatch at n_seq = 1) against
one UnicornSOTTrack per target plus one UnicornMOTTracker, bit for bit on every frame (detections, counts, priors, raw head outputs,
MOT boxes / ids / NMS rows / embeddings or ByteTrack tracks)."""
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

TINY = (320, 320)
FULL = (800, 1280)
STEPS = 22
ADD = {"a": (0, 0), "b": (3, 1), "c": (7, 2)}  # target id -> (frame it is added on, object of make_video)
REMOVE = {"b": 12}  # target id -> first frame it is no longer tracked on
MOT_KW = dict(conf=0.01, nms=0.7, score_thr=0.02)


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


def video(size, n=STEPS, seed=40):
    from unicorn_b200.synthetic import make_video
    return make_video(n, *size, seed=seed, n_obj=6)


def qd_tracker():
    from unicorn_b200.tracker import QuasiDenseEmbedTracker
    # seeded weights give low scores: lower the score gates so that tracklets are created (as tests/test_mot_batch_gpu.py)
    return QuasiDenseEmbedTracker(init_score_thr=0.05, obj_score_thr=0.03)


def byte_tracker():
    from unicorn_b200.tracker import BYTETracker
    from unicorn_b200.tracker.byte_tracker import STrack
    STrack._count = 0  # track ids are a class-wide counter: each run starts from the same one
    return BYTETracker(types.SimpleNamespace(track_thresh=0.05, track_buffer=30, match_thresh=0.9, mot20=False))


def new_tracker(mot):
    return {"qd": qd_tracker, "byte": byte_tracker, None: lambda: None}[mot]()


def byte_rows(tracks):
    return np.array([[t.track_id, *t.tlwh, t.score] for t in tracks], dtype=np.float64).reshape(-1, 6)


# ------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("act", [0, 1, 3])
def test_zero_table_gather_matches_groupnorm_apply(act):
    from unicorn_b200 import ops, shared_ops
    g = torch.Generator(device="cuda").manual_seed(1)
    h, w, C, G_, n_plain, n_prior = 12, 20, 256, 16, 2, 3
    wide = torch.randn(1, h, w, C + 64, device="cuda", generator=g).bfloat16()
    x = wide[..., 32:32 + C]  # a channel slice: pixel stride C + 64
    x[0, 0] = -300.0  # with the large weights below, SiLU of these pixels is -0.0 in the images without a prior
    st = torch.zeros(G_, 2, dtype=torch.int64, device="cuda")
    xs = x.float().reshape(h * w, G_, C // G_)
    fix = 1 << 22
    st[:, 0] = (xs.sum(dim=(0, 2)) * fix).round().long()
    st[:, 1] = ((xs * xs).sum(dim=(0, 2)) * fix).round().long()
    gw = torch.randn(C, device="cuda", generator=g)
    gw[:16] = 100.0
    gb = torch.randn(C, device="cuda", generator=g)
    beta = torch.randn(C, device="cuda", generator=g)
    prior = torch.rand(n_prior, 1, h, w, device="cuda", generator=g)
    prior[1] = 0.0  # a zero prior plane still takes the prior path, as its own B = 1 call does
    out = torch.full((n_plain + n_prior, h, w, C), 7.0, dtype=torch.bfloat16, device="cuda")
    zeros = torch.zeros(n_plain + n_prior, dtype=torch.int32, device="cuda")  # every image reads the one source image
    shared_ops.groupnorm_apply_gather(x, st, gw, gb, G_, 1e-3, act, out, n_plain, zeros, prior=prior.reshape(-1), beta=beta)
    for b in range(n_plain + n_prior):
        ref = torch.empty(1, h, w, C, dtype=torch.bfloat16, device="cuda")
        pr = prior[b - n_plain].reshape(-1).contiguous() if b >= n_plain else None
        ops.groupnorm_apply(x, st, gw, gb, G_, 1e-3, act, out=ref, prior=pr, beta=beta if pr is not None else None)
        same(out[b:b + 1], ref, f"image {b}")
    # the no-prior images keep their negative zeros (adding a zero prior would make them +0)
    if act == 3:
        assert (bits(out[:n_plain]) == -32768).any()


# ------------------------------------------------------------------------------------------------ engine
@pytest.mark.parametrize("mot", [True, False])
@pytest.mark.parametrize("K", [1, 3])
def test_head_shared_matches_head_per_image(K, mot):
    e = engine("unicorn_track_tiny")
    frames, _ = video(TINY, n=1)
    g = torch.Generator(device="cuda").manual_seed(2)
    e.begin_frame()
    fpn, _ = e.backbone(frames[:1].cuda())
    priors = [torch.rand(K, 1, f.shape[1], f.shape[2], device="cuda", generator=g) for f in fpn]
    got_mot, got_sot = e.head_shared(fpn, priors, mot=mot)
    got_mot = got_mot.clone() if mot else None
    got_sot = got_sot.clone()
    assert got_sot.shape[0] == K and (got_mot is None or got_mot.shape[-1] == 5 + e.ncls)
    if mot:
        same(got_mot, e.head(fpn, None, "mot"), "mot image")
    for k in range(K):
        same(got_sot[k:k + 1], e.head(fpn, [p[k] for p in priors], "sot"), f"sot image {k}")


def test_head_shared_one_class_mot_head():
    """unicorn_track_large_mot_challenge: a 1-class MOT head next to 1-class SOT heads, each decoded into its own buffer."""
    e = engine("unicorn_track_large_mot_challenge")
    frames, _ = video(TINY, n=1)
    g = torch.Generator(device="cuda").manual_seed(3)
    assert e.ncls == 1
    for K in (1, 2):
        e.begin_frame()
        fpn, _ = e.backbone(frames[:1].cuda())
        priors = [torch.rand(K, 1, f.shape[1], f.shape[2], device="cuda", generator=g) for f in fpn]
        got_mot, got_sot = (t.clone() for t in e.head_shared(fpn, priors))
        same(got_mot, e.head(fpn, None, "mot"), f"K {K} mot image")
        for k in range(K):
            same(got_sot[k:k + 1], e.head(fpn, [p[k] for p in priors], "sot"), f"K {K} sot image {k}")


# ------------------------------------------------------------------------------------------------ driver
def sot_reference(e, size, frames, boxes, tid):
    """UnicornSOTTrack initialised on the target's reference frame: {frame: (dets, count, priors, head)}."""
    from unicorn_b200.sot import UnicornSOTTrack
    f0, obj = ADD[tid]
    stop = REMOVE.get(tid, len(frames))
    trk = UnicornSOTTrack(e, size)
    trk.initialize_tensor(frames[f0:f0 + 1], boxes[f0, obj])
    out = {}
    for t in range(f0 + 1, stop):
        dets, n = trk.track_tensor(frames[t:t + 1])
        out[t] = (dets.clone(), n, [p.reshape(-1).cpu() for p in trk.last["priors"]], trk.last["head"].cpu())
    return out


def mot_reference(e, size, frames, mot, kw):
    from unicorn_b200.mot import UnicornMOTTracker
    trk = UnicornMOTTracker(e, size, tracker=new_tracker(mot), assoc=mot, use_graph=True, **kw)
    out = []
    for t in range(len(frames)):
        res = trk.step_tensor(frames[t:t + 1], img_info=size)
        res = byte_rows(res) if mot == "byte" else (res[0].clone(), res[1].clone())
        feats = trk.last["feats"].clone() if mot == "qd" else None
        out.append((res, trk.last["dets"].clone(), feats, trk.last["head"].cpu()))
    return out


def run_unified(e, size, frames, boxes, mot, kw, max_targets, use_graph=True, pipelined=False):
    """UnicornUnifiedTracker over `frames` with the ADD / REMOVE schedule: per frame (results, last_dets, last_feats, priors, heads)."""
    from unicorn_b200.unified import UnicornUnifiedTracker
    trk = UnicornUnifiedTracker(e, size, max_targets, mot=mot, tracker=new_tracker(mot), mot_conf=kw["conf"], mot_nms=kw["nms"],
                                score_thr=kw["score_thr"], use_graph=use_graph)
    out, graphs = [], []

    def schedule(t):
        for tid, (f0, obj) in ADD.items():
            if f0 == t:
                trk.add_target(tid, boxes[t, obj])
        for tid, f1 in REMOVE.items():
            if f1 == t:
                trk.remove_target(tid)

    def record(res):
        if mot == "byte":
            res["mot"] = byte_rows(res["mot"])
        slots = {t: i for i, t in enumerate(trk._tid)}
        extra = {tid: ([p.reshape(trk.max_targets, -1)[slots[tid]].cpu() for p in trk.last["priors"]],
                       trk.last["head_sot"][slots[tid]].cpu()) for tid in res["targets"] if tid in slots}
        mh = trk.last["head_mot"].cpu() if mot is not None else None
        out.append((res, trk.last_dets, trk.last_feats, extra, mh))
        graphs.append(trk.graph)

    if not pipelined:
        for t in range(len(frames)):
            schedule(t)
            record(trk.step_tensor(frames[t:t + 1], img_info=size))
    else:  # submit(t + 1) before collect(t): only the host values of the step are compared (the device buffers are step t + 1's)
        schedule(0)
        trk.submit(frames[0:1])
        for t in range(len(frames)):
            if t + 1 < len(frames):
                schedule(t + 1)
                trk.submit(frames[t + 1:t + 2])
            res = trk.collect(size)
            if mot == "byte":
                res["mot"] = byte_rows(res["mot"])
            out.append((res, trk.last_dets, trk.last_feats, None, None))
    return out, graphs


def check_against_references(e, size, mot, max_targets, n=STEPS, kw=MOT_KW):
    frames, boxes = video(size, n=n)
    sot = {tid: sot_reference(e, size, frames, boxes, tid) for tid in ADD}
    ref_mot = mot_reference(e, size, frames, mot, kw) if mot is not None else None
    got, graphs = run_unified(e, size, frames, boxes, mot, kw, max_targets)
    n_dets = 0
    for t, (res, dets, feats, extra, head_mot) in enumerate(got):
        live = {tid for tid in ADD if ADD[tid][0] < t < REMOVE.get(tid, n)}
        assert set(res["targets"]) == live, (t, set(res["targets"]), live)
        for tid in live:
            rd, rn, rpri, rhead = sot[tid][t]
            gd, gn = res["targets"][tid]
            assert gn == rn, (t, tid, gn, rn)
            same(gd, rd, f"frame {t} target {tid} dets")
            gpri, ghead = extra[tid]
            for lvl in range(3):
                same(gpri[lvl], rpri[lvl], f"frame {t} target {tid} prior {lvl}")
            same(ghead, rhead[0], f"frame {t} target {tid} head")
            n_dets += rn
        if mot is None:
            assert res["mot"] is None
            continue
        rres, rdets, rfeats, rhead = ref_mot[t]
        same(head_mot, rhead, f"frame {t} MOT head")
        same(dets, rdets, f"frame {t} NMS rows")
        if mot == "qd":
            same(feats, rfeats, f"frame {t} embeddings")
            same(res["mot"][0], rres[0], f"frame {t} boxes")
            assert torch.equal(res["mot"][1], rres[1]), (t, res["mot"][1], rres[1])
        else:
            assert np.array_equal(res["mot"], rres), (t, res["mot"], rres)
    assert n_dets > 0, "no SOT detections: a vacuous test"
    if mot is not None:
        assert any(r[1].shape[0] > 0 for r in ref_mot), "no MOT detections: a vacuous test"
    # first step eager, second captured; targets added on frames 3 and 7 and removed on frame 12 keep that graph
    assert graphs[0] is None and graphs[1] is not None and all(g is graphs[1] for g in graphs[1:])
    return frames, boxes, got


@pytest.mark.parametrize("mot", ["qd", "byte", None])
def test_unified_tiny_matches_separate_drivers(mot):
    e = engine("unicorn_track_tiny")
    frames, boxes, got = check_against_references(e, TINY, mot, max_targets=4)  # slot 3 is never used: always one free slot
    # graph equals eager, and the pipelined protocol (submit(t + 1) before collect(t)) gives the same results
    eager, _ = run_unified(e, TINY, frames, boxes, mot, MOT_KW, 4, use_graph=False, pipelined=True)
    for t, (a, b) in enumerate(zip(got, eager)):
        assert a[0]["targets"].keys() == b[0]["targets"].keys(), t
        for tid in a[0]["targets"]:
            same(a[0]["targets"][tid][0], b[0]["targets"][tid][0], f"frame {t} target {tid}")
            assert a[0]["targets"][tid][1] == b[0]["targets"][tid][1]
        if mot is not None:
            same(a[1], b[1], f"frame {t} NMS rows")
        if mot == "qd":
            same(a[0]["mot"][0], b[0]["mot"][0], f"frame {t} boxes")
            assert torch.equal(a[0]["mot"][1], b[0]["mot"][1])
        elif mot == "byte":
            assert np.array_equal(a[0]["mot"], b[0]["mot"]), t


@pytest.mark.parametrize("mot", ["qd", "byte", None])
def test_unified_large_full_size_matches_separate_drivers(mot):
    check_against_references(engine("unicorn_track_large"), FULL, mot, max_targets=3)


def test_unified_r50_matches_separate_drivers():
    check_against_references(engine("unicorn_track_r50"), TINY, "qd", max_targets=3, n=14)


def test_free_slot_contents_do_not_change_other_targets():
    """A free slot computes on whatever its buffers hold: garbage there changes no other target's result."""
    from unicorn_b200.unified import UnicornUnifiedTracker
    e = engine("unicorn_track_tiny")
    frames, boxes = video(TINY, n=4)
    runs = []
    for garbage in (False, True):
        trk = UnicornUnifiedTracker(e, TINY, 2, mot=None)
        trk.add_target("a", boxes[0, 0])
        trk.step_tensor(frames[0:1])
        if garbage:
            trk.ref_proj[0][trk.ref_proj[0].shape[0] // 2:].normal_()
            trk.ref_proj[1][trk.ref_proj[1].shape[0] // 2:].normal_()
            trk.lbs_pre[1].uniform_()
        runs.append([trk.step_tensor(frames[t:t + 1])["targets"] for t in range(1, 4)])
        assert trk.sot_ws.count[1].item() == 0  # the free slot's count is zeroed on the device
    for a, b in zip(*runs):
        assert a.keys() == b.keys() == {"a"}
        same(a["a"][0], b["a"][0])


def test_reference_protocol_matches_separate_drivers():
    """track(image, new_targets) letterboxes once: its states equal UnicornSOTTrack.track's, its MOT output UnicornMOTTracker's."""
    from unicorn_b200.mot import UnicornMOTTracker
    from unicorn_b200.sot import UnicornSOTTrack, preprocess
    from unicorn_b200.unified import UnicornUnifiedTracker
    e = engine("unicorn_track_tiny")
    frames, boxes = video((240, 400), n=6)  # letterboxed into 320x320: r = 0.8
    imgs = [f.permute(1, 2, 0).flip(-1).round().to(torch.uint8).numpy().copy() for f in frames]  # RGB HWC
    xywh = lambda b: [float(b[0]), float(b[1]), float(b[2] - b[0]), float(b[3] - b[1])]  # noqa: E731
    sot = UnicornSOTTrack(e, TINY)
    sot.initialize(imgs[1], {"init_bbox": xywh(boxes[1, 0])})
    ref_states = {t: sot.track(imgs[t])["target_bbox"] for t in range(2, 6)}
    mtrk = UnicornMOTTracker(e, TINY, tracker=qd_tracker(), use_graph=True, **MOT_KW)
    ref_mot = []
    for im in imgs:
        f, r = preprocess(im, TINY)
        b, i = mtrk.step_tensor(f, r, img_info=im.shape[:2])
        ref_mot.append((b.clone(), i.clone()))
    trk = UnicornUnifiedTracker(e, TINY, 2, mot="qd", tracker=qd_tracker(), mot_conf=MOT_KW["conf"], mot_nms=MOT_KW["nms"],
                                score_thr=MOT_KW["score_thr"])
    for t, im in enumerate(imgs):
        out = trk.track(im, new_targets={"a": xywh(boxes[1, 0])} if t == 1 else None)
        if t == 0:
            assert out["targets"] == {}
        elif t == 1:
            assert out["targets"] == {"a": xywh(boxes[1, 0])}
        else:
            assert out["targets"] == {"a": ref_states[t]}, t
        same(out["mot"][0], ref_mot[t][0], f"frame {t} boxes")
        assert torch.equal(out["mot"][1], ref_mot[t][1])


def test_rejections_change_nothing():
    from unicorn_b200.unified import UnicornUnifiedTracker
    e = engine("unicorn_track_tiny")
    frames, boxes = video(TINY, n=2)
    with pytest.raises(ValueError, match="mot must be"):
        UnicornUnifiedTracker(e, TINY, 2, mot="sort")
    with pytest.raises(ValueError, match="BYTETracker"):
        UnicornUnifiedTracker(e, TINY, 2, mot="byte")
    trk = UnicornUnifiedTracker(e, TINY, 2, mot=None)
    trk.add_target("a", boxes[0, 0])
    with pytest.raises(ValueError, match="duplicate"):
        trk.add_target("a", boxes[0, 1])
    trk.add_target("b", boxes[0, 1])
    with pytest.raises(ValueError, match="exceed max_targets"):
        trk.add_target("c", boxes[0, 2])
    with pytest.raises(ValueError, match="unknown target"):
        trk.remove_target("c")
    with pytest.raises(ValueError, match="frame must be"):
        trk.submit(frames[0:1, :, :160])
    with pytest.raises(ValueError, match="duplicate"):
        trk.track(np.zeros((320, 320, 3), np.uint8), new_targets={"a": [0, 0, 10, 10]})
    assert trk.targets == ["a", "b"] and trk._ring.submitted == 0 and sorted(trk._pending) == [0, 1]


def test_detector_config_is_rejected():
    from unicorn_b200.unified import UnicornUnifiedTracker
    e = engine("unicorn_det_convnext_tiny")
    with pytest.raises(ValueError, match="detector"):
        UnicornUnifiedTracker(e, TINY, 1)

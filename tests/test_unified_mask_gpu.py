"""One backbone pass per frame for VOS objects and a MOTS arm: the shared-trunk head with the controllers against head(..., with_masks=True)
at B = 1, and UnicornUnifiedMaskTracker against one UnicornVOSTrack plus one UnicornMOTSTracker, bit for bit on every frame (object
rows, counts and masks, label map, soft masks, MOTS ids / RLE strings / NMS rows / embeddings)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

TINY = (320, 320)
FULL = (800, 1280)
STEPS = 20
FIRST = {1: 0, 2: 1}  # objects added on frame 0 without a mask: object id -> object of make_video
LATER = (3, {3: 2})   # frame, objects added on it with an init_mask
REMOVE = (12, 2)      # frame before whose submit the object is removed, object id
MOTS_KW = dict(mots_conf=0.01, mots_nms=0.7, score_thr=0.02, max_dets=16, min_box_area=300)  # the lowered gates of test_mots_batch_gpu


def bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else (torch.uint8 if t.element_size() == 1 else torch.int32))


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


def qd_tracker():
    from unicorn_b200.tracker import QuasiDenseEmbedTracker
    return QuasiDenseEmbedTracker(init_score_thr=0.05, obj_score_thr=0.03)


def u8(frames):
    return frames.round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()


def label_map(box, oid, H, W):
    lab = torch.zeros(H, W, dtype=torch.uint8)
    x1, y1, x2, y2 = box.round().int().tolist()
    lab[max(y1, 0):max(y2, 0), max(x1, 0):max(x2, 0)] = oid
    return lab


class Video:
    """n letterboxed uint8 frames [n,H,W,3] of an original size, the objects' boxes in resized-image and original coordinates."""

    def __init__(self, size, orig, n, seed=40):
        from unicorn_b200.sot import preprocess
        from unicorn_b200.synthetic import make_video
        frames, boxes = make_video(n, *orig, seed=seed, n_obj=3)
        self.size, self.orig = size, tuple(orig)
        if tuple(orig) == tuple(size):
            self.frames, self.r = u8(frames), 1.0
        else:
            rgb = [f.permute(1, 2, 0).flip(-1).round().clamp(0, 255).to(torch.uint8).numpy().copy() for f in frames]
            lb = [preprocess(im, size) for im in rgb]
            self.frames, self.r = torch.cat([f.clone() for f, _ in lb]), lb[0][1]
        self.orig_boxes, self.boxes = boxes, boxes * self.r

    def init_mask(self, t, objs):
        lab = torch.zeros(self.orig, dtype=torch.uint8)
        for oid, o in objs.items():
            m = label_map(self.orig_boxes[t, o], oid, *self.orig)
            lab[m > 0] = oid
        return lab


def snap(vos, counts):
    """A VOS result dict copied to the host, with each object's detection count."""
    return dict(seg=vos["segmentation"].cpu().clone(), soft=vos["soft"].cpu().clone(), ids=list(vos["ids"]), counts=dict(counts),
                objects={k: (None if d is None else d.clone(), None if m is None else m.cpu().clone()) for k, (d, m) in vos["objects"].items()})


def same_vos(a, b, what, objs=None):
    """a and b agree on the objects `objs` (default all); with all objects also on the ids, label map and soft masks."""
    keys = a["objects"].keys() if objs is None else objs
    if objs is None:
        assert a["ids"] == b["ids"], (what, a["ids"], b["ids"])
        assert a["objects"].keys() == b["objects"].keys(), what
        same(a["seg"], b["seg"], what + " segmentation")
        same(a["soft"], b["soft"], what + " soft")
    for k in keys:
        (d, m), (d2, m2) = a["objects"][k], b["objects"][k]
        assert a["counts"][k] == b["counts"][k], (what, k, a["counts"][k], b["counts"][k])
        assert (d is None) == (d2 is None), (what, k)
        if d is not None:
            same(d, d2, f"{what} object {k} row")
            same(m, m2, f"{what} object {k} mask")


def vos_reference(e, v, n):
    """One UnicornVOSTrack: FIRST on frame 0, LATER with its init_mask; {frame: snap}."""
    from unicorn_b200.vos import UnicornVOSTrack
    trk = UnicornVOSTrack(e, v.size, use_graph=True)
    trk.initialize_tensor(v.frames[0:1], {oid: v.boxes[0, o] for oid, o in FIRST.items()}, orig_size=v.orig, r=v.r)
    out = {}
    for t in range(1, n):
        if t == LATER[0]:
            res = trk.track_tensor(v.frames[t:t + 1], {oid: v.boxes[t, o] for oid, o in LATER[1].items()}, v.init_mask(t, LATER[1]))
        else:
            res = trk.track_tensor(v.frames[t:t + 1])
        s = trk._workers[0]
        counts = {oid: int(s.rows_host[po["slot"], 7]) for oid, po in s.last["per_obj"].items()}
        out[t] = snap(res, counts)
    return out


def mots_reference(e, v, n):
    """One UnicornMOTSTracker: per frame (write_results_mots tuple, NMS rows, embeddings)."""
    from unicorn_b200.mots import UnicornMOTSTracker
    kw = {k.replace("mots_", ""): val for k, val in MOTS_KW.items()}
    trk = UnicornMOTSTracker(e, v.size, tracker=qd_tracker(), use_graph=True, **kw)
    out = []
    for t in range(n):
        res = trk.step_tensor(v.frames[t:t + 1], *v.orig)
        out.append((res, trk.last["dets"].clone(), trk.last["feats"].clone()))
    return out


def run_unified(e, v, n, mots, use_graph=True, pipelined=False, remove=None, max_objects=4, max_groups=3):
    """UnicornUnifiedMaskTracker over the first n frames with the FIRST / LATER (/ remove) schedule: per frame (vos snap, mots tuple,
    NMS rows, embeddings), and the parity graphs after every step."""
    from unicorn_b200.unified import UnicornUnifiedMaskTracker
    trk = UnicornUnifiedMaskTracker(e, v.size, v.orig, max_objects, max_groups, mots=mots, tracker=qd_tracker() if mots else None,
                                    use_graph=use_graph, **MOTS_KW)
    out, graphs = [], []

    def schedule(t):
        if t == 0:
            trk.add_objects({oid: v.boxes[0, o] for oid, o in FIRST.items()})
        if t == LATER[0]:
            trk.add_objects({oid: v.boxes[t, o] for oid, o in LATER[1].items()}, init_mask=v.init_mask(t, LATER[1]))
        if remove is not None and t == remove[0]:
            trk.remove_object(remove[1])

    def record(res):
        counts = {oid: int(row[7]) for oid, row in trk.last_rows.items()}
        out.append((snap(res["vos"], counts), res["mots"], trk.last_dets, trk.last_feats))
        graphs.append(trk.graphs)

    if not pipelined:
        for t in range(n):
            schedule(t)
            record(trk.step_tensor(v.frames[t:t + 1]))
    else:  # submit(t + 1) before collect(t)
        schedule(0)
        trk.submit(v.frames[0:1])
        for t in range(n):
            if t + 1 < n:
                schedule(t + 1)
                trk.submit(v.frames[t + 1:t + 2])
            record(trk.collect())
    return trk, out, graphs


def check_against_references(e, v, n, mots, remove=None):
    ref_vos = vos_reference(e, v, n)
    ref_mots = mots_reference(e, v, n) if mots else None
    trk, got, graphs = run_unified(e, v, n, mots, remove=remove)
    assert got[0][0]["ids"] == [] and not got[0][0]["seg"].any(), "frame 0 is the reference frame of the first objects"
    n_dets = n_enc = 0
    for t in range(1, n):
        g, want = got[t][0], ref_vos[t]
        if remove is None or t < remove[0]:
            same_vos(g, want, f"frame {t}")
        else:  # the remaining objects equal VOSTrack's, the label map is the aggregate of their masks
            from unicorn_b200 import ops
            keep = [o for o in want["ids"] if o != remove[1]]
            assert g["ids"] == keep and set(g["objects"]) == set(keep), (t, g["ids"])
            same_vos(g, want, f"frame {t}", objs=keep)
            H0, W0 = v.orig
            seg = torch.zeros(H0, W0, dtype=torch.uint8, device="cuda")
            soft = torch.zeros(len(keep), H0, W0, device="cuda")
            masks = [(m if m is not None else torch.zeros(v.size)).cuda()[None].contiguous() for _, m in (want["objects"][o] for o in keep)]
            ops.vos_aggregate(masks, None, keep, *v.size, v.r, soft, seg)
            same(g["seg"], seg.cpu(), f"frame {t} segmentation after the removal")
            same(g["soft"], soft.cpu(), f"frame {t} soft after the removal")
        n_dets += sum(c > 0 for c in g["counts"].values())
        if not mots:
            assert got[t][1] is None
            continue
    if mots:
        for t in range(n):
            rres, rdets, rfeats = ref_mots[t]
            assert got[t][1] == rres, (t, got[t][1], rres)
            same(got[t][2], rdets, f"frame {t} NMS rows")
            same(got[t][3], rfeats, f"frame {t} embeddings")
            n_enc += len(rres[5])
        assert n_enc > 0, "no MOTS instance was encoded: a vacuous test"
    assert n_dets > 0, "no VOS detections: a vacuous test"
    assert got[-1][0]["seg"].max() > 0
    # the first step runs eagerly, each parity slot's next step is captured; adding and removing objects never re-captures
    assert graphs[0] == [None, None] and graphs[1][0] is None and graphs[1][1] is not None
    assert all(g[0] is graphs[2][0] and g[1] is graphs[2][1] for g in graphs[2:]) and graphs[2][0] is not None
    return got


# ------------------------------------------------------------------------------------------------ engine
def check_head_shared_with_masks(e, Ks, mots):
    from unicorn_b200.synthetic import make_video
    frames, _ = make_video(1, *TINY, seed=40)
    g = torch.Generator(device="cuda").manual_seed(2)
    for K in Ks:
        e.begin_frame()
        fpn, _ = e.backbone(frames[:1].cuda())
        priors = [torch.rand(K, 1, f.shape[1], f.shape[2], device="cuda", generator=g) for f in fpn]
        got_mot, got_sot = e.head_shared(fpn, priors, mot=mots, with_masks=True)
        got_mot = got_mot.clone() if mots else None
        got_sot = got_sot.clone()
        dyn = [t.clone() for t in e.dyn_levels]
        n_mot = int(mots)
        assert all(t.shape[0] == n_mot + K and t.shape[-1] == 176 for t in dyn)
        if mots:
            same(got_mot, e.head(fpn, None, "mot", with_masks=True), f"K {K} mot image")
            for lvl in range(3):
                same(dyn[lvl][:1], e.dyn_levels[lvl], f"K {K} mot image controllers {lvl}")
        for k in range(K):
            same(got_sot[k:k + 1], e.head(fpn, [p[k] for p in priors], "sot", with_masks=True), f"K {K} sot image {k}")
            for lvl in range(3):
                same(dyn[lvl][n_mot + k:n_mot + k + 1], e.dyn_levels[lvl], f"K {K} sot image {k} controllers {lvl}")


@pytest.mark.parametrize("mots", [True, False])
def test_head_shared_with_masks_matches_head_per_image(mots):
    check_head_shared_with_masks(engine("unicorn_track_tiny_mask"), (1, 3), mots)


def test_head_shared_with_masks_one_class_mot_head():
    e = engine("unicorn_track_large_mot_challenge_mask")
    assert e.ncls == 1
    check_head_shared_with_masks(e, (1, 2), True)


# ------------------------------------------------------------------------------------------------ driver
@pytest.mark.parametrize("mots", [True, False])
def test_unified_mask_tiny_matches_separate_drivers(mots):
    e = engine("unicorn_track_tiny_mask")
    v = Video(TINY, TINY, STEPS)
    got = check_against_references(e, v, STEPS, mots, remove=REMOVE)
    # eager equals graph, and the pipelined protocol (submit(t + 1) before collect(t)) equals the sequential one; the object removed
    # before submit(12) is still reported by step 11, which was submitted before the removal
    for use_graph in (False, True):
        _, other, _ = run_unified(e, v, STEPS, mots, use_graph=use_graph, pipelined=True, remove=REMOVE)
        for t, (a, b) in enumerate(zip(got, other)):
            same_vos(a[0], b[0], f"use_graph={use_graph} pipelined frame {t}")
            assert a[1] == b[1], t
            if mots:
                same(a[2], b[2], f"frame {t} NMS rows")
                same(a[3], b[3], f"frame {t} embeddings")
    assert got[REMOVE[0] - 1][0]["ids"] == [1, 2, 3] and got[REMOVE[0]][0]["ids"] == [1, 3]


def test_unified_mask_large_full_size_matches_separate_drivers():
    """unicorn_track_large_mask at 800x1280 from 1080x1920 frames (r = 2/3)."""
    check_against_references(engine("unicorn_track_large_mask"), Video(FULL, (1080, 1920), 6, seed=41), 6, True)


def test_unified_mask_r50_matches_separate_drivers():
    check_against_references(engine("unicorn_track_r50_mask"), Video(TINY, TINY, 8, seed=42), 8, True)


def test_free_slot_contents_do_not_change_live_objects():
    """Free object and group slots compute on whatever their buffers hold: garbage there changes no live result."""
    from unicorn_b200.unified import UnicornUnifiedMaskTracker
    e = engine("unicorn_track_tiny_mask")
    v = Video(TINY, TINY, 5, seed=43)
    runs = []
    for garbage in (False, True):
        trk = UnicornUnifiedMaskTracker(e, TINY, TINY, 2, 2, mots=True, tracker=qd_tracker(), **MOTS_KW)
        trk.add_objects({1: v.boxes[0, 0]})
        trk.step_tensor(v.frames[0:1])
        if garbage:
            n = trk.ref_proj[0].shape[0] // 2
            trk.ref_proj[0][n:].normal_()
            trk.ref_proj[1][n:].normal_()
            trk.lbs[1].uniform_()
            trk.obj_row[1].fill_(trk.R + 1)  # the free object slot reads a row of the free group slot
        res = []
        for t in range(1, 5):
            out = trk.step_tensor(v.frames[t:t + 1])
            res.append((snap(out["vos"], {o: int(r[7]) for o, r in trk.last_rows.items()}), out["mots"]))
            assert trk.vos_ws.count[1].item() == 0  # the free slot's count is zeroed on the device
            assert not trk._ring.slots[t % 2].vos_masks[1].any()
        runs.append(res)
    for t, (a, b) in enumerate(zip(*runs)):
        assert a[0]["ids"] == [1]
        same_vos(a[0], b[0], f"frame {t + 1}")
        assert a[1] == b[1]


def test_reference_protocol_matches_separate_drivers():
    """track(image, info) letterboxes once: its label maps and states equal UnicornVOSTrack.track's, its MOTS tuples those of
    UnicornMOTSTracker.step_tensor on the same letterboxed frames."""
    from unicorn_b200.mots import UnicornMOTSTracker
    from unicorn_b200.sot import preprocess
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.unified import UnicornUnifiedMaskTracker
    from unicorn_b200.vos import UnicornVOSTrack
    e = engine("unicorn_track_tiny_mask")
    orig = (240, 400)  # letterboxed into 320x320: r = 0.8
    frames, boxes = make_video(6, *orig, seed=44, n_obj=3)
    imgs = [f.permute(1, 2, 0).flip(-1).round().clamp(0, 255).to(torch.uint8).numpy().copy() for f in frames]  # RGB HWC
    xywh = lambda b: [float(b[0]), float(b[1]), float(b[2] - b[0]), float(b[3] - b[1])]  # noqa: E731
    first = {"init_object_ids": ["1", "2"], "init_bbox": {"1": xywh(boxes[0, 0]), "2": xywh(boxes[0, 1])}}
    lab = label_map(boxes[3, 2], 3, *orig).numpy()
    later = {"init_object_ids": ["3"], "init_bbox": {"3": xywh(boxes[3, 2])}, "init_mask": lab}
    vos = UnicornVOSTrack(e, TINY, use_graph=True)
    vos.initialize(imgs[0], first)
    ref, states = {}, {}
    for t in range(1, 6):
        ref[t] = vos.track(imgs[t], later if t == 3 else None)["segmentation"]
        states[t] = dict(vos.state_pre_dict)
    kw = {k.replace("mots_", ""): val for k, val in MOTS_KW.items()}
    mtrk = UnicornMOTSTracker(e, TINY, tracker=qd_tracker(), use_graph=True, **kw)
    ref_mots = [mtrk.step_tensor(preprocess(im, TINY)[0], *orig) for im in imgs]
    trk = UnicornUnifiedMaskTracker(e, TINY, orig, 3, 2, tracker=qd_tracker(), **MOTS_KW)
    for t, im in enumerate(imgs):
        out = trk.track(im, first if t == 0 else later if t == 3 else None)
        assert out["mots"] == ref_mots[t], t
        if t == 0:
            assert not out["segmentation"].any() and trk.state_pre_dict == {k: first["init_bbox"][k] for k in ("1", "2")}
            continue
        assert np.array_equal(out["segmentation"], ref[t]), t
        assert trk.state_pre_dict == states[t], t
    assert out["segmentation"].max() > 0


def test_rejections_change_nothing():
    from unicorn_b200.unified import UnicornUnifiedMaskTracker
    e = engine("unicorn_track_tiny_mask")
    v = Video(TINY, TINY, 2, seed=45)
    trk = UnicornUnifiedMaskTracker(e, TINY, TINY, 4, 3, mots=False)
    trk.add_objects({1: v.boxes[0, 0], 2: v.boxes[0, 1]})

    def state():
        return (list(trk.objects), [(list(b), m is None) for b, m in trk._b._pending[0]], list(trk._b._os), list(trk._b._gs), trk._ring.submitted,
                trk.frame_id, trk.active.tolist(), trk.obj_row.tolist())
    before = state()
    good_mask = torch.zeros(TINY, dtype=torch.uint8)
    with pytest.raises(ValueError, match="duplicate"):
        trk.add_objects({1: v.boxes[0, 2]})
    with pytest.raises(ValueError, match="duplicate"):
        trk.add_objects({4: v.boxes[0, 2], "4": v.boxes[0, 2]})
    with pytest.raises(ValueError, match="1..255"):
        trk.add_objects({0: v.boxes[0, 2]})
    with pytest.raises(ValueError, match="3 new objects but 2 of max_objects = 4 slots are free"):
        trk.add_objects({4: v.boxes[0, 2], 5: v.boxes[0, 2], 6: v.boxes[0, 2]})
    with pytest.raises(ValueError, match="4 values"):
        trk.add_objects({4: [0.0, 1.0, 2.0]})
    with pytest.raises(ValueError, match="init_mask"):
        trk.add_objects({4: v.boxes[0, 2]}, init_mask=torch.zeros(160, 320, dtype=torch.uint8))
    with pytest.raises(ValueError, match="init_mask"):
        trk.add_objects({4: v.boxes[0, 2]}, init_mask=torch.zeros(TINY, dtype=torch.int64))
    with pytest.raises(ValueError, match="unknown object"):
        trk.remove_object(7)
    with pytest.raises(ValueError, match="frame must be"):
        trk.submit(v.frames[0:1, :160])
    with pytest.raises(ValueError, match="has size"):
        trk.track(np.zeros((240, 400, 3), np.uint8))
    assert state() == before
    trk.add_objects({3: v.boxes[0, 2]}, init_mask=good_mask)
    before = state()
    with pytest.raises(ValueError, match="already has an init_mask"):
        trk.add_objects({4: v.boxes[0, 2]}, init_mask=good_mask)
    assert state() == before
    trk.add_objects({4: v.boxes[0, 2]})  # the third group slot: all are taken now
    before = state()
    trk2 = UnicornUnifiedMaskTracker(e, TINY, TINY, 4, 3, mots=False)
    with pytest.raises(ValueError, match="max_groups"):
        for oid in range(1, 5):
            trk2.add_objects({oid: v.boxes[0, 0]})
    assert trk2.objects == [1, 2, 3] and trk2._b._gs == [1, 1, 1]
    big = UnicornUnifiedMaskTracker(e, TINY, TINY, 17, 3, mots=False)
    with pytest.raises(ValueError, match="at most 16"):
        big.add_objects({o: v.boxes[0, 0] for o in range(1, 18)})
    assert big.objects == [] and big._b._gs == [0, 0, 0] and big._b._os == [None] * 17
    # the driver still runs on the state it had: frame 0 is the reference of objects 1..4, object 3 enters from its (empty) mask
    assert state() == before
    res = trk.step_tensor(v.frames[0:1])
    assert res["vos"]["ids"] == [3] and res["mots"] is None and trk.objects == [1, 2, 3, 4]
    assert trk._b.image_of.tolist() == [0, 0, 0, 0]  # the reference frame made every object slot live: it reads video 0's image
    trk.step_tensor(v.frames[1:2])
    assert trk.active.tolist() == [1, 1, 1, 1]  # the step's active table


@pytest.mark.parametrize("name", ["unicorn_track_tiny", "unicorn_det_convnext_tiny"])
def test_configs_without_the_tracking_mask_head_are_rejected(name):
    from unicorn_b200.unified import UnicornUnifiedMaskTracker
    e = engine(name)
    with pytest.raises(ValueError, match="mask"):
        UnicornUnifiedMaskTracker(e, TINY, TINY, 1)
    if not e.det:
        e.begin_frame()
        from unicorn_b200.synthetic import make_video
        fpn, _ = e.backbone(make_video(1, *TINY, seed=0)[0].cuda())
        prior = [torch.zeros(1, f.shape[1], f.shape[2], device="cuda") for f in fpn]
        with pytest.raises(ValueError, match="no mask head"):
            e.head_shared(fpn, prior, with_masks=True)

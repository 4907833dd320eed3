"""Batched VOS (B > 1) against the same images and sequences run one at a time, bit for bit: the batched mask kernels, the
correlation's rows against its row count, the mask branch and masked head of the engine (eager and as one CUDA graph), and the
multi-sequence VOS driver UnicornVOSBatch against one UnicornVOSTrack per sequence.  UnicornVOSTrack is held to the reference class
and to per-launch fp32 references by the other test files; batching must not change a single bit of what it computes."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))


def G(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def same(a, b, what=""):
    assert a.shape == b.shape, (what, a.shape, b.shape)
    assert torch.equal(a, b), (what, (a.float() - b.float()).abs().max().item())


def u8(frames):
    """fp32 BGR [n,3,H,W] (synthetic.make_video) -> the uint8 [n,H,W,3] frames the drivers stage."""
    return frames.round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()


# ------------------------------------------------------------------------------------------------ kernels
def test_aligned_bilinear_add_batched():
    from unicorn_b200 import ops
    B, hs, ws, C = 3, 10, 16, 128
    for f in (2, 4):
        src = torch.randn(B, hs, ws, C, device="cuda", generator=G(f)).bfloat16()
        dst0 = torch.randn(B, hs * f, ws * f, C, device="cuda", generator=G(10 + f)).bfloat16()
        got = ops.aligned_bilinear_add(src, dst0.clone(), f)
        for b in range(B):
            same(got[b:b + 1], ops.aligned_bilinear_add(src[b:b + 1].contiguous(), dst0[b:b + 1].clone(), f), f"factor {f} image {b}")


def test_dynamic_masks_batched():
    """Four head images on two mask-branch images: counts 0, 1, more than n_max and 2; image_of maps two heads to image 1 and one
    entry out of range (that head image is skipped: nothing written, nothing read)."""
    from unicorn_b200 import ops
    h, w, up, d, n_max = 16, 20, 4, 2, 3
    hw = [(16, 20), (8, 10), (4, 5)]
    A = sum(a * b for a, b in hw)
    S, B = 2, 4
    mf = torch.randn(S, h, w, 8, device="cuda", generator=G(1))
    um = torch.randn(S, h, w, 9 * up * up, device="cuda", generator=G(2))
    dyn = [torch.randn(B, a, b, 176, device="cuda", generator=G(3 + k)) * 0.3 for k, (a, b) in enumerate(hw)]
    ws = ops.PostWorkspace(A, "cuda", B)
    ws.count.copy_(torch.tensor([0, 1, 5, 2], dtype=torch.int32))
    ws.anchors.copy_(torch.randint(0, A, (B, A), device="cuda", generator=G(7), dtype=torch.int32))
    image_of = torch.tensor([1, 1, 5, 0], dtype=torch.int32, device="cuda")
    out = ops.dynamic_masks(mf, um, dyn, hw, ws, n_max, up_rate=up, d_rate=d, image_of=image_of)
    assert out.shape == (B, n_max, h * up * d, w * up * d)
    for b in range(B):
        img = int(image_of[b])
        if not 0 <= img < S:
            assert not out[b].any(), "a skipped head image was written"
            continue
        ws1 = ops.PostWorkspace(A, "cuda")
        ws1.count.copy_(ws.count[b:b + 1])
        ws1.anchors.copy_(ws.anchors[b])
        ref = ops.dynamic_masks(mf[img:img + 1].contiguous(), um[img:img + 1].contiguous(), [t[b:b + 1].contiguous() for t in dyn], hw, ws1, n_max,
                                up_rate=up, d_rate=d)
        same(out[b], ref, f"head image {b}")
    assert out[2].abs().sum() == 0 and out[1, 0].any() and out[0].abs().sum() == 0
    # identity mapping without image_of (S = B) and d_rate 1
    mf4, um4 = mf.repeat(2, 1, 1, 1), um.repeat(2, 1, 1, 1)
    out4 = ops.dynamic_masks(mf4, um4, dyn, hw, ws, n_max, up_rate=up, d_rate=1)
    for b in (1, 3):
        ws1 = ops.PostWorkspace(A, "cuda")
        ws1.count.copy_(ws.count[b:b + 1])
        ws1.anchors.copy_(ws.anchors[b])
        ref = ops.dynamic_masks(mf4[b:b + 1].contiguous(), um4[b:b + 1].contiguous(), [t[b:b + 1].contiguous() for t in dyn], hw, ws1, n_max,
                                up_rate=up, d_rate=1)
        same(out4[b], ref, f"identity image {b}")


def test_corr_rows_do_not_depend_on_row_count():
    """Rows 0..k-1 of an R-row correlation equal a k-row launch: a group slot may carry more label rows than its group has objects."""
    from unicorn_b200 import ops
    Gs, n_ref, n_cur = 2, 1600, 1600
    K = torch.randn(Gs, n_ref, 128, device="cuda", generator=G(1)).half()
    Q = torch.randn(Gs, n_cur, 128, device="cuda", generator=G(2)).half()
    V = torch.rand(Gs, 8, n_ref, device="cuda", generator=G(3))
    for R in (8, 4, 2):
        full = ops.corr_propagate(K, Q, V[:, :R].contiguous())
        for k in range(1, R):
            part = ops.corr_propagate(K, Q, V[:, :k].contiguous())
            same(full[:, :k], part, f"R={R} k={k}")
            same(full[0, :k], ops.corr_propagate(K[0], Q[0], V[0, :k].contiguous()), f"R={R} k={k} unbatched")


# ------------------------------------------------------------------------------------------------ engine
def mask_frame(e, imgs, priors, tag):
    e.begin_frame()
    feats, _ = e.features(imgs, tag)
    fpn = e.neck(feats, tag)
    mf, um = e.mask_branch(fpn)
    head = e.head(fpn, priors, "sot", with_masks=True)
    out = dict(mf=mf, um=um, head=head, dyn0=e.dyn_levels[0], dyn1=e.dyn_levels[1], dyn2=e.dyn_levels[2])
    return {k: v.clone() for k, v in out.items()}


def check_mask_batch(e, B, H, W, seed):
    from unicorn_b200.synthetic import make_video
    frames, _ = make_video(B, H, W, seed=seed)
    imgs = frames.cuda().contiguous()
    priors = [torch.rand(B, H // s, W // s, device="cuda", generator=G(seed + s)) for s in (8, 16, 32)]
    ones = [mask_frame(e, imgs[b:b + 1], [p[b:b + 1] for p in priors], "m1") for b in range(B)]
    eager = mask_frame(e, imgs, priors, "mb")
    for b in range(B):
        for k, v in ones[b].items():
            same(eager[k][b:b + 1], v, f"B={B} image {b} {k}")
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    res = {}
    with torch.cuda.graph(g):
        res.update(mask_frame(e, imgs, priors, "mb"))
    g.replay()
    torch.cuda.synchronize()
    for k, v in eager.items():
        same(res[k], v, f"graph {k}")


@pytest.fixture(scope="module")
def tiny():
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.weights import make_state_dict
    return UnicornEngine(make_state_dict("unicorn_track_tiny_mask", 0), "unicorn_track_tiny_mask")


def test_engine_mask_path_batched_tiny(tiny):
    check_mask_batch(tiny, 3, 320, 320, seed=4)


@pytest.fixture(scope="module")
def large():
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.weights import make_state_dict
    return UnicornEngine(make_state_dict("unicorn_track_large_mask", 0), "unicorn_track_large_mask")


def test_engine_mask_path_batched_fullsize(large):
    check_mask_batch(large, 3, 800, 1280, seed=6)


# ------------------------------------------------------------------------------------------------ driver
def snap(o):
    """A result dict of track_tensor, copied to the host."""
    if o is None:
        return None
    return dict(seg=o["segmentation"].cpu().clone(), soft=o["soft"].cpu().clone(), ids=list(o["ids"]),
                objects={k: (None if d is None else d.clone(), None if m is None else m.cpu().clone()) for k, (d, m) in o["objects"].items()})


def same_result(a, b, what):
    assert (a is None) == (b is None), what
    if a is None:
        return
    assert a["ids"] == b["ids"], (what, a["ids"], b["ids"])
    same(a["seg"], b["seg"], what + " segmentation")
    same(a["soft"], b["soft"], what + " soft")
    assert a["objects"].keys() == b["objects"].keys(), what
    for k, (d, m) in a["objects"].items():
        d2, m2 = b["objects"][k]
        assert (d is None) == (d2 is None), (what, k)
        if d is not None:
            same(d, d2, f"{what} object {k} row")
            same(m, m2, f"{what} object {k} mask")


def label_map(box, oid, H, W):
    lab = torch.zeros(H, W, dtype=torch.uint8)
    x1, y1, x2, y2 = box.int().tolist()
    lab[y1:y2, x1:x2] = oid
    return lab


def scenario(n_frames=9):
    """Four synthetic sequences and their events, per slot of a 4-slot batch:
      slot 0: sequence A (1 object) until step 4, then re-initialised with sequence D (2 objects) on D's frame 4;
      slot 1: sequence B (2 objects) that gains object 3 at step 3 (a new reference group);
      slot 2: sequence C (3 objects), idle at steps 5 and 6;
      slot 3: never initialised."""
    from unicorn_b200.synthetic import make_video
    vids = {k: make_video(n_frames, 320, 320, seed=40 + s, n_obj=3) for s, k in enumerate("ABCD")}
    return {k: (u8(f), b) for k, (f, b) in vids.items()}


def run_single(eng, frames, boxes, ids, start, steps, new_at=None, use_graph=False):
    from unicorn_b200.vos import UnicornVOSTrack
    t = UnicornVOSTrack(eng, (320, 320), use_graph=use_graph)
    t.initialize_tensor(frames[start:start + 1], {o: boxes[start, o - 1] for o in ids})
    out = {}
    for f in steps:
        if f == new_at:
            out[f] = snap(t.track_tensor(frames[f:f + 1], {3: boxes[f, 2]}, label_map(boxes[f, 2], 3, 320, 320)))
        else:
            out[f] = snap(t.track_tensor(frames[f:f + 1]))
    return out


def run_batch(eng, vids, use_graph, n_frames=9):
    from unicorn_b200.vos import UnicornVOSBatch
    vb = UnicornVOSBatch(eng, (320, 320), 4, max_objects=8, max_groups=4, use_graph=use_graph)
    fa, ba = vids["A"]
    fb, bb = vids["B"]
    fc, bc = vids["C"]
    fd, bd = vids["D"]
    vb.initialize_tensor(0, fa[0:1], {1: ba[0, 0]})
    vb.initialize_tensor(1, fb[0:1], {1: bb[0, 0], 2: bb[0, 1]})
    vb.initialize_tensor(2, fc[0:1], {1: bc[0, 0], 2: bc[0, 1], 3: bc[0, 2]})
    steps = []
    for f in range(1, n_frames):
        if f == 4:
            vb.initialize_tensor(0, fd[4:5], {1: bd[4, 0], 2: bd[4, 1]})
            continue  # the re-initialisation consumes D's frame 4; nothing else advances in this step
        frames = [fd[f:f + 1] if f > 4 else fa[f:f + 1], fb[f:f + 1], None if f in (5, 6) else fc[f:f + 1], fa[f:f + 1]]
        new = {1: ({3: bb[f, 2]}, label_map(bb[f, 2], 3, 320, 320))} if f == 3 else None
        steps.append((f, [snap(o) for o in vb.track_tensor(frames, new)]))
    return vb, steps


def test_vos_batch_equals_separate_trackers(tiny):
    eng = tiny
    vids = scenario()
    fa, ba = vids["A"]
    fb, bb = vids["B"]
    fc, bc = vids["C"]
    fd, bd = vids["D"]
    want = {0: run_single(eng, fa, ba, [1], 0, [1, 2, 3]), 1: run_single(eng, fb, bb, [1, 2], 0, [1, 2, 3, 5, 6, 7, 8], new_at=3),
            2: run_single(eng, fc, bc, [1, 2, 3], 0, [1, 2, 3, 7, 8]), "D": run_single(eng, fd, bd, [1, 2], 4, [5, 6, 7, 8])}
    outs = {}
    for use_graph in (True, False):
        _, steps = run_batch(eng, vids, use_graph)
        outs[use_graph] = steps
        for f, res in steps:
            assert res[3] is None, "slot 3 was never initialised"
            for i in range(3):
                what = f"graph={use_graph} step {f} slot {i}"
                if i == 2 and f in (5, 6):
                    assert res[i] is None, what
                    continue
                ref = want["D"][f] if (i == 0 and f > 4) else want[i][f]
                same_result(res[i], ref, what)
        last = dict(steps)[8]
        assert last[1]["ids"] == [1, 2, 3] and last[0]["ids"] == [1, 2]
    for (f, a), (_, b) in zip(outs[True], outs[False]):  # graph replay equals eager
        for i in range(4):
            same_result(a[i], b[i], f"graph vs eager step {f} slot {i}")


def test_vos_batch_reference_protocol_golden(tiny):
    """The reference-protocol fixture of test_vos_gpu in slot 1 of a two-slot batch: label maps equal UnicornVOSTrack's."""
    from make_golden_vos_common import make_sequence
    from unicorn_b200.vos import UnicornVOSBatch, UnicornVOSTrack
    g = np.load(os.path.join(ROOT, "tests", "golden", "vos_tiny.npz"))
    assert str(g["config"]) == "unicorn_track_tiny_mask"
    size, new_at, n = tuple(int(v) for v in g["size"]), int(g["new_at"]), int(g["n_frames"])
    rgb, xywh, lab = make_sequence()
    init = {"init_object_ids": ["1", "2"], "sequence_object_ids": ["1", "2", "3"],
            "init_bbox": {"1": xywh[0, 0].tolist(), "2": xywh[0, 1].tolist()}}
    other = {"init_object_ids": ["5"], "init_bbox": {"5": xywh[1, 1].tolist()}}
    trk = UnicornVOSTrack(tiny, size, use_graph=True)
    trk.initialize(rgb[0], init)
    vb = UnicornVOSBatch(tiny, size, 2, max_objects=4, max_groups=3)
    vb.initialize(0, rgb[1], other)
    vb.initialize(1, rgb[0], init)
    for t in range(1, n):
        info = {"init_object_ids": ["3"], "init_bbox": {"3": xywh[t, 2].tolist()}, "init_mask": lab} if t == new_at else {}
        want = trk.track(rgb[t], info)["segmentation"]
        got = vb.track([rgb[n - t], rgb[t]], [None, info])
        assert np.array_equal(got[1]["segmentation"], want), t
        assert got[0] is not None and got[0]["segmentation"].shape == want.shape
        assert vb.state_pre_dicts[1] == trk.state_pre_dict, t
    assert got[1]["segmentation"].max() <= 3


def test_vos_batch_fullsize(large):
    """unicorn_track_large_mask at 800x1280: a 3-object and a 1-object sequence equal two UnicornVOSTracks."""
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.vos import UnicornVOSBatch, UnicornVOSTrack
    H, W = 800, 1280
    vids = [make_video(4, H, W, seed=60 + s, n_obj=3) for s in range(2)]
    vids = [(u8(f), b) for f, b in vids]
    objs = [[1, 2, 3], [2]]
    vb = UnicornVOSBatch(large, (H, W), 2, max_objects=4, max_groups=2)
    want = []
    for i, ((fr, bx), ids) in enumerate(zip(vids, objs)):
        t = UnicornVOSTrack(large, (H, W), use_graph=True)
        t.initialize_tensor(fr[0:1], {o: bx[0, o - 1] for o in ids})
        want.append([snap(t.track_tensor(fr[f:f + 1])) for f in range(1, 4)])
        vb.initialize_tensor(i, fr[0:1], {o: bx[0, o - 1] for o in ids})
    for f in range(1, 4):
        got = vb.track_tensor(torch.cat([fr[f:f + 1] for fr, _ in vids]))
        for i in range(2):
            same_result(snap(got[i]), want[i][f - 1], f"frame {f} sequence {i}")


def test_vos_batch_capacity(tiny):
    """Requests beyond max_objects, max_groups or 16 objects per sequence raise ValueError and change nothing."""
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.vos import UnicornVOSBatch
    fr, bx = make_video(4, 320, 320, seed=70, n_obj=3)
    fr = u8(fr)

    def fresh():
        vb = UnicornVOSBatch(tiny, (320, 320), 3, max_objects=3, max_groups=2)
        vb.initialize_tensor(0, fr[0:1], {1: bx[0, 0], 2: bx[0, 1]})
        return vb
    ref = fresh()
    want = [snap(o) for o in ref.track_tensor(torch.cat([fr[1:2]] * 3))]
    vb = fresh()
    with pytest.raises(ValueError, match="max_objects"):
        vb.initialize_tensor(1, fr[0:1], {1: bx[0, 0], 2: bx[0, 1]})  # 4 objects > max_objects = 3
    vb.initialize_tensor(1, fr[0:1], {1: bx[0, 2]})  # 2 groups, 3 objects: full
    with pytest.raises(ValueError, match="max_groups|max_objects"):
        vb.initialize_tensor(2, fr[0:1], {1: bx[0, 2]})
    with pytest.raises(ValueError, match="max_groups|max_objects"):
        vb.track_tensor(torch.cat([fr[1:2]] * 3), {0: ({3: bx[1, 2]}, label_map(bx[1, 2], 3, 320, 320))})
    assert vb.seqs[2] is None and vb.seqs[0].obj_ids == [1, 2]
    got = [snap(o) for o in vb.track_tensor(torch.cat([fr[1:2]] * 3))]
    same_result(got[0], want[0], "slot 0 after the refused requests")
    assert got[2] is None
    big = UnicornVOSBatch(tiny, (320, 320), 1, max_objects=20, max_groups=4)
    with pytest.raises(ValueError, match="at most 16"):
        big.initialize_tensor(0, fr[0:1], {o: bx[0, 0] for o in range(1, 18)})
    assert big.seqs[0] is None

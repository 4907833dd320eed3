"""Batched frames (B > 1) against the same images run one at a time (B = 1), bit for bit: the batched kernels, every engine stage
eager and as one CUDA graph, engine reuse across batch sizes, the multi-sequence SOT driver and the model API.  The B = 1 path is
held to the oracle and to per-launch fp32 references by the other test files; batching must not change a single bit of it."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))


def G(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def same(a, b, what=""):
    assert a.shape == b.shape, (what, a.shape, b.shape)
    assert torch.equal(a, b), (what, (a.float() - b.float()).abs().max().item())


# ------------------------------------------------------------------------------------------------ kernels
def test_flat_conv_groupnorm_stats_per_image():
    """1x1 stride-1 conv with GroupNorm statistics on 3 distinct images: each image's sums land in its own slot (the flat layout used
    to fold the batch into one row and add every image's sums to image 0's)."""
    from unicorn_b200 import ops
    B, H, W, Cin, Cout, Gr = 3, 20, 24, 64, 128, 16
    x = (torch.randn(B, H, W, Cin, device="cuda", generator=G(0)) * (1 + torch.arange(B, device="cuda")[:, None, None, None])).bfloat16()
    w = ops.pack_conv_weight(torch.randn(Cout, Cin, 1, 1, device="cuda", generator=G(1)) * 0.1)
    st = torch.zeros(B, Gr, 2, dtype=torch.int64, device="cuda")
    y = ops.conv2d(x, w, 1, 1, out=torch.empty(B, H, W, Cout, dtype=torch.bfloat16, device="cuda"), gn_stats=st, gn_groups=Gr)
    for b in range(B):
        st1 = torch.zeros(Gr, 2, dtype=torch.int64, device="cuda")
        y1 = ops.conv2d(x[b:b + 1].contiguous(), w, 1, 1, gn_stats=st1, gn_groups=Gr)
        same(y[b:b + 1], y1, f"y{b}")
        same(st[b], st1, f"stats{b}")
    assert not torch.equal(st[0], st[1])


def test_msda_fused_batched():
    from unicorn_b200 import ops
    B, lv, M, P = 3, [(10, 12), (10, 12)], 8, 4
    n = 120
    vals = [torch.randn(2 * n, 256, device="cuda", generator=G(10 + b)).bfloat16() for b in range(B)]
    offs = [torch.randn(2 * n, 192, device="cuda", generator=G(20 + b)) * 2 for b in range(B)]
    # rows [level][image][pixel]
    value = torch.cat([v[l * n:(l + 1) * n] for l in range(2) for v in vals]).contiguous()
    offlog = torch.cat([o[l * n:(l + 1) * n] for l in range(2) for o in offs]).contiguous()
    out = ops.msda_fused(value, offlog, lv, M, P)
    for b in range(B):
        ref = ops.msda_fused(vals[b], offs[b], lv, M, P)
        for l in range(2):
            same(out[(l * B + b) * n:(l * B + b + 1) * n], ref[l * n:(l + 1) * n], f"image {b} level {l}")


@pytest.mark.parametrize("n_obj", [1, 3])
def test_corr_propagate_batched(n_obj):
    from unicorn_b200 import ops
    B, n_ref, n_cur = 3, 1000, 900
    K = torch.randn(B, n_ref, 128, device="cuda", generator=G(1)).half()
    Q = torch.randn(B, n_cur, 128, device="cuda", generator=G(2)).half()
    V = torch.rand(B, n_obj, n_ref, device="cuda", generator=G(3))
    out = ops.corr_propagate(K, Q, V)
    for b in range(B):
        same(out[b], ops.corr_propagate(K[b], Q[b], V[b].contiguous()), f"sequence {b}")


@pytest.mark.parametrize("ncls", [1, 8])
def test_head_decode_batched(ncls):
    from unicorn_b200 import ops
    B, hw = 3, [(16, 20), (8, 10), (4, 5)]
    ro = [torch.randn(B, h, w, 8, device="cuda", generator=G(k)) for k, (h, w) in enumerate(hw)]
    cl = [torch.randn(B, h, w, 8, device="cuda", generator=G(10 + k)) for k, (h, w) in enumerate(hw)]
    out = ops.head_decode(ro, cl, hw, (8, 16, 32), ncls)
    for b in range(B):
        same(out[b:b + 1], ops.head_decode([t[b:b + 1] for t in ro], [t[b:b + 1] for t in cl], hw, (8, 16, 32), ncls), f"image {b}")


@pytest.mark.parametrize("ncls", [1, 8])
@pytest.mark.parametrize("max_keep", [0, 3])
def test_postprocess_batched(ncls, max_keep):
    """Three images in one launch sequence, the middle one with no detection at all."""
    from unicorn_b200 import ops
    B, A = 3, 2100
    g = G(ncls * 10 + max_keep)
    pred = torch.empty(B, A, 5 + ncls, device="cuda")
    pred[..., :2] = torch.rand(B, A, 2, device="cuda", generator=g) * 300
    pred[..., 2:4] = torch.rand(B, A, 2, device="cuda", generator=g) * 60 + 4
    pred[..., 4:] = torch.rand(B, A, 1 + ncls, device="cuda", generator=g)
    pred[1, :, 4] = 0.0
    ws = ops.PostWorkspace(A, "cuda", B)
    dets, cnt = ops.postprocess_device(pred, ncls, 0.3, 0.45, ws, max_keep=max_keep)
    torch.cuda.synchronize()
    assert dets.shape == (B, A, 7) and cnt.shape == (B,)
    assert int(cnt[1]) == 0 and int(cnt[0]) > 0 and int(cnt[2]) > 0
    for b in range(B):
        ws1 = ops.PostWorkspace(A, "cuda")
        d1, c1 = ops.postprocess_device(pred[b].contiguous(), ncls, 0.3, 0.45, ws1, max_keep=max_keep)
        n = int(c1[0])
        assert int(cnt[b]) == n, (b, int(cnt[b]), n)
        same(dets[b, :n], d1[:n], f"dets {b}")
        same(ws.anchors[b, :n], ws1.anchors[:n], f"anchors {b}")
        if max_keep:
            assert n <= max_keep


# ------------------------------------------------------------------------------------------------ engine
def sot_frame(e, imgs, refs, values):
    """One SOT frame of len(imgs) sequences on the engine's stages (imgs fp32 [B,3,H,W], refs the reference frames, values the label
    values [B, 1, n8]); returns every stage's output as a clone."""
    from unicorn_b200 import ops
    B = imgs.shape[0]
    e.begin_frame()
    fr, sr = e.features(refs, "bref")
    e.neck(fr, "bref")
    feat0 = sr["feat"].clone()
    e.begin_frame()
    feats, seq = e.features(imgs, "bcur")
    fpn = e.neck(feats, "bcur")
    f0, f1 = e.interaction(feat0, seq["feat"])
    e0, e1 = e.upsample(f0, "bemb0"), e.upsample(f1, "bemb1")
    pri = e.propagate(e0, e1, values if B > 1 else values[0])
    head = e.head(fpn, pri, "sot")
    H, W = imgs.shape[2:]
    ws = ops.PostWorkspace(head.shape[1], e.dev, B)
    d, c = ops.postprocess_device(head, 1, 0.001, 0.65, ws, max_keep=3)
    out = dict(fpn0=fpn[0], fpn1=fpn[1], fpn2=fpn[2], feat=seq["feat"], f0=f0, f1=f1, e0=e0, e1=e1, pri0=pri[0], pri1=pri[1],
               pri2=pri[2], head=head, dets=d.view(B, -1, 7)[:, :3], count=c)
    return {k: v.clone() for k, v in out.items()}


def split(o, b):
    """Image b of a batched result, shaped like a B = 1 result."""
    r = {}
    for k, v in o.items():
        if k.startswith("pri"):
            r[k] = v[b]
        else:
            r[k] = v[b:b + 1]
    return r


def check_batch(eng, B, H, W, seed):
    from unicorn_b200.synthetic import make_video
    frames, boxes = make_video(2 * B, H, W, seed=seed)
    imgs, refs = frames[B:].cuda().contiguous(), frames[:B].cuda().contiguous()
    values = torch.rand(B, 1, (H // 8) * (W // 8), device="cuda", generator=G(seed))
    ones = [sot_frame(eng, imgs[b:b + 1], refs[b:b + 1], values[b:b + 1]) for b in range(B)]
    eager = sot_frame(eng, imgs, refs, values)
    for b in range(B):
        got = split(eager, b)
        for k, v in ones[b].items():
            if k == "dets":
                n = min(int(ones[b]["count"][0]), 3)  # rows past the count are stale workspace
                same(got[k][:, :n], v[:, :n], f"B={B} image {b} {k}")
            else:
                same(got[k].reshape(v.shape), v, f"B={B} image {b} {k}")
    # the batched frame as one CUDA graph (every buffer already exists)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    res = {}
    with torch.cuda.graph(g):
        res.update(sot_frame(eng, imgs, refs, values))
    g.replay()
    torch.cuda.synchronize()
    for k, v in eager.items():
        if k == "dets":
            for b in range(B):
                n = min(int(eager["count"][b]), 3)
                same(res[k][b, :n], v[b, :n], f"graph dets {b}")
        else:
            same(res[k], v, f"graph {k}")
    return eager


@pytest.fixture(scope="module")
def tiny():
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.weights import make_state_dict
    sd = make_state_dict("unicorn_track_tiny", 0)
    return sd, UnicornEngine(sd, "unicorn_track_tiny")


def test_engine_stages_batched_tiny(tiny):
    check_batch(tiny[1], 3, 320, 320, seed=3)


@pytest.mark.parametrize("name", ["unicorn_track_large", "unicorn_track_r50"])
def test_engine_stages_batched_fullsize(name):
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.weights import make_state_dict
    eng = UnicornEngine(make_state_dict(name, 0), name)
    check_batch(eng, 2, 800, 1280, seed=5)


def test_engine_reuse_across_batch_sizes(tiny):
    """A B = 1 frame after B = 4 frames on one engine equals a fresh engine's."""
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.synthetic import make_video
    sd, eng = tiny
    frames, _ = make_video(8, 320, 320, seed=9)
    values = torch.rand(4, 1, 1600, device="cuda", generator=G(9))
    for _ in range(2):
        sot_frame(eng, frames[4:].cuda().contiguous(), frames[:4].cuda().contiguous(), values)
    got = sot_frame(eng, frames[4:5].cuda().contiguous(), frames[0:1].cuda().contiguous(), values[:1])
    ref = sot_frame(UnicornEngine(sd, "unicorn_track_tiny"), frames[4:5].cuda().contiguous(), frames[0:1].cuda().contiguous(), values[:1])
    for k, v in ref.items():
        same(got[k], v, k)


# ------------------------------------------------------------------------------------------------ multi-sequence SOT driver
def rgb(frame):
    """fp32 BGR [3,H,W] (synthetic.make_video) -> the RGB HWC uint8 frame a user hands to track()."""
    return frame.permute(1, 2, 0).flip(-1).round().to(torch.uint8).contiguous()


@pytest.fixture(scope="module")
def videos():
    from unicorn_b200.synthetic import make_video
    return [make_video(8, 320, 320, seed=20 + s) for s in range(4)]


def single(eng, frames, boxes, start, stop, use_graph=True):
    from unicorn_b200.sot import UnicornSOTTrack
    t = UnicornSOTTrack(eng, (320, 320), use_graph=use_graph)
    t.initialize_tensor(frames[start:start + 1], boxes[start, 0])
    return [t.track_tensor(frames[f:f + 1]) for f in range(start + 1, stop)]


def test_sot_batch_equals_separate_trackers(tiny, videos):
    from unicorn_b200.sot import UnicornSOTBatch
    eng = tiny[1]
    refs = [single(eng, fr, bx, 0, 8) for fr, bx in videos]
    fresh2 = single(eng, *videos[2], 4, 8)  # slot 2 re-initialised on its frame 4
    outs = {}
    for use_graph in (True, False):
        sb = UnicornSOTBatch(eng, (320, 320), 4, use_graph=use_graph)
        for i, (fr, bx) in enumerate(videos):
            sb.initialize_tensor(i, fr[0:1], bx[0, 0])
        steps = []
        for f in range(1, 8):
            if f == 5:
                sb.initialize_tensor(2, videos[2][0][4:5], videos[2][1][4, 0])
            steps.append(sb.track_tensor(torch.stack([fr[f] for fr, _ in videos])))
        outs[use_graph] = steps
        for s, (dets, counts) in enumerate(steps):
            f = s + 1
            for i in range(4):
                want_d, want_n = fresh2[f - 5] if (i == 2 and f >= 5) else refs[i][s]
                assert int(counts[i]) == want_n, (use_graph, f, i, int(counts[i]), want_n)
                same(dets[i, :want_d.shape[0]], want_d, f"graph={use_graph} frame {f} slot {i}")
    for (d0, c0), (d1, c1) in zip(outs[True], outs[False]):  # graph replay equals eager
        same(c0, c1)
        for i in range(4):
            same(d0[i, :min(int(c0[i]), 3)], d1[i, :min(int(c1[i]), 3)])


def test_sot_batch_idle_slot(tiny, videos):
    from unicorn_b200.sot import UnicornSOTBatch, UnicornSOTTrack
    eng = tiny[1]
    sb = UnicornSOTBatch(eng, (320, 320), 4, device_preproc=True)
    sep = []
    for i, (fr, bx) in enumerate(videos):
        t = UnicornSOTTrack(eng, (320, 320), device_preproc=True)
        init = {"init_bbox": [float(v) for v in (bx[0, 0, 0], bx[0, 0, 1], bx[0, 0, 2] - bx[0, 0, 0], bx[0, 0, 3] - bx[0, 0, 1])]}
        t.initialize(rgb(fr[0]).numpy(), init)
        sb.initialize(i, rgb(fr[0]).numpy(), init)
        sep.append(t)
    for f in range(1, 6):
        idle = 1 if f in (2, 3) else None
        res = sb.track([None if i == idle else rgb(fr[f]).numpy() for i, (fr, _) in enumerate(videos)])
        for i, (fr, _) in enumerate(videos):
            if i == idle:
                assert res[i] is None
                continue
            assert res[i] == sep[i].track(rgb(fr[f]).numpy()), (f, i)


# ------------------------------------------------------------------------------------------------ model API
def test_shim_batched_equals_single(tiny):
    import unicorn_oracle as orc
    from unicorn_b200.compat.model import UnicornB200Model, postprocess
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.weights import make_state_dict
    g = np.load(os.path.join(ROOT, "tests", "golden", "whole_tiny_320.npz"))
    frames, _ = make_video(2, 320, 320, seed=int(g["seed_video"]), n_obj=int(g["n_obj"]))
    f = int(g["frame"])
    imgs = torch.stack([frames[1 - f], frames[f]]).cuda().contiguous()  # the golden frame at batch index 1
    model = UnicornB200Model(tiny[0], "unicorn_track_tiny").eval()
    head2, seq2 = model(imgs=imgs, mode="whole")
    head2 = head2.clone()
    feat2 = seq2["feat"].clone()
    ones = [model(imgs=imgs[b:b + 1], mode="whole") for b in range(2)]
    ones = [(h.clone(), s["feat"].clone()) for h, s in ones]
    for b in range(2):
        same(head2[b:b + 1], ones[b][0], f"head {b}")
        same(feat2[b:b + 1], ones[b][1], f"feat {b}")
    # the golden image at batch index 1 meets the fixture's tolerances (tests/test_whole_gpu.py)
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from test_whole_gpu import check_dets, check_head
    check_head(head2[1:2], g["head"])
    dets2 = postprocess(head2.clone(), 8, float(g["conf"]), float(g["nms"]))
    for b in range(2):
        d1 = postprocess(ones[b][0].clone(), 8, float(g["conf"]), float(g["nms"]))[0]
        assert (d1 is None) == (dets2[b] is None)
        if d1 is not None:
            same(dets2[b], d1, f"dets {b}")
    check_dets(dets2[1].cpu(), g["dets"], orc)
    # interaction / upsample
    _, sa = model(imgs=imgs, mode="backbone")
    sa = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in sa.items()}
    _, sb = model(imgs=imgs.flip(0).contiguous(), mode="backbone")
    sb = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in sb.items()}
    f0, f1 = (t.clone() for t in model(seq_dict0=sa, seq_dict1=sb, mode="interaction"))
    up = model(feat=f1, mode="upsample").clone()
    for b in range(2):
        d0 = dict(sa, feat=sa["feat"][b:b + 1])
        d1 = dict(sb, feat=sb["feat"][b:b + 1])
        g0, g1 = model(seq_dict0=d0, seq_dict1=d1, mode="interaction")
        same(f0[b:b + 1], g0, f"interaction feat0 {b}")
        same(f1[b:b + 1], g1, f"interaction feat1 {b}")
        same(up[b:b + 1], model(feat=g1.clone(), mode="upsample"), f"upsample {b}")


def test_mask_config_rejects_batches():
    from unicorn_b200.compat.model import UnicornB200Model
    from unicorn_b200.weights import make_state_dict
    model = UnicornB200Model(make_state_dict("unicorn_track_tiny_mask", 0), "unicorn_track_tiny_mask").eval()
    imgs = torch.rand(2, 3, 320, 320, device="cuda") * 255
    with pytest.raises(ValueError, match="one image"):
        model(imgs=imgs, mode="whole")
    fpn, _ = model(imgs=imgs, mode="backbone")
    with pytest.raises(ValueError, match="one image"):
        model.head(fpn, None, mode="mot")

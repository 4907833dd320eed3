"""uc_mots_encode against the host restatement (F.interpolate + threshold + results.overlap_free + results.rle_encode), the MOTS
driver's submit / collect with CUDA graphs against its sequential protocol and mots_frame_result, and the MOTS Challenge model
(unicorn_track_large_mot_challenge_mask) against the oracle."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
HIN, WIN, THR = 800, 1280, 0.3
SIZES = [(1080, 1920), (480, 640), (720, 1280), (402, 640)]  # 720 x 1280: r = 1; 402 x 640: 401 rows (short masks)


def ratio(h, w):
    return min(HIN / float(h), WIN / float(w))


def resized(masks, order, r, h, w):
    return F.interpolate(masks[order.long()][:, None], scale_factor=1 / r, mode="bilinear", align_corners=False)[:, 0, :h, :w]


def reference(masks, order, emit, r, h, w):
    from unicorn_b200 import results as R
    if order.numel() == 0:
        return [], None
    v = resized(masks, order, r, h, w)
    free = R.overlap_free(v > THR).cpu().numpy()
    return [R.rle_encode(free[i]) if emit[i] else "" for i in range(order.numel())], v


def blob_masks(n, seed):
    """0 / 1 masks: ellipses, plus an empty mask (row 0), a full mask (row 1), one covering pixel (0, 0) (row 2) and one touching the
    bottom and right edges (row 3)."""
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.arange(HIN, dtype=torch.float32), torch.arange(WIN, dtype=torch.float32), indexing="ij")
    out = torch.zeros(n, HIN, WIN)
    for i in range(4, n):
        cy, cx = (torch.rand(2, generator=g) * torch.tensor([HIN, WIN])).tolist()
        ay, ax = (30 + torch.rand(2, generator=g) * torch.tensor([HIN / 4, WIN / 4])).tolist()
        out[i] = (((yy - cy) / ay) ** 2 + ((xx - cx) / ax) ** 2 < 1).float()
    out[1] = 1.0
    out[2, :90, :150] = 1.0
    out[3, int(HIN * 0.7):, int(WIN * 0.6):] = 1.0
    return out.cuda()


def order_and_emit(k, n_max, seed):
    """k mask rows: the special rows first (the full mask second to last), every fifth instance not emitted."""
    g = torch.Generator().manual_seed(seed)
    rest = [i for i in torch.randperm(n_max, generator=g).tolist() if i > 3]
    rows = [2, 3, 0] + rest
    rows = rows[:k] if k < 4 else rows[:k - 2] + [1] + rows[k - 2:k - 1]
    emit = [i % 5 != 4 for i in range(k)]
    return torch.tensor(rows, dtype=torch.int32), emit


def run(enc, masks, order, emit, r, h, w):
    return enc(masks, order.tolist(), emit, THR, r, h, w)


@pytest.fixture(scope="module")
def blobs():
    return blob_masks(64, 0)


@pytest.mark.parametrize("k", [0, 1, 20, 64])
@pytest.mark.parametrize("size", SIZES)
def test_encode_is_byte_identical_to_the_host_path(blobs, size, k):
    from unicorn_b200.mots import MaskEncoder
    h, w = size
    r = ratio(h, w)
    order, emit = order_and_emit(k, 64, k)
    want, v = reference(blobs, order, emit, r, h, w)
    if v is not None:
        assert ((v - THR).abs() < 1e-6).sum().item() == 0  # inputs far from the threshold: the strings must be identical
    got = run(MaskEncoder(64, "cuda"), blobs, order, emit, r, h, w)
    assert got == want


@pytest.mark.parametrize("size", SIZES)
def test_encode_smooth_random_masks_differ_only_at_the_threshold(size):
    """Continuous masks have pixels at the threshold, where the resize may round differently: decoded masks may differ only at
    pixels within 1e-5 of thr (in this instance or an earlier one, which hides it)."""
    from unicorn_b200 import results as R
    from unicorn_b200.mots import MaskEncoder
    h, w = size
    r = ratio(h, w)
    g = torch.Generator().manual_seed(h)
    masks = F.interpolate(torch.rand(24, 1, HIN // 40, WIN // 40, generator=g), size=(HIN, WIN), mode="bilinear",
                          align_corners=False)[:, 0].contiguous().cuda()
    order = torch.randperm(24, generator=g)[:20].to(torch.int32)
    emit = [True] * 20
    want, v = reference(masks, order, emit, r, h, w)
    got = run(MaskEncoder(24, "cuda"), masks, order, emit, r, h, w)
    hm, wm = v.shape[1:]
    near = (((v - THR).abs() < 1e-5).cumsum(0) > 0).cpu()
    flips = 0
    for i in range(20):
        if got[i] == want[i]:
            continue
        diff = torch.from_numpy(R.rle_decode(got[i], hm, wm) ^ R.rle_decode(want[i], hm, wm))
        assert not (diff & ~near[i]).any(), f"instance {i}: a pixel away from the threshold differs"
        flips += int(diff.sum())
    print(f"{size}: {flips} pixels differ, {int(near[-1].sum())} within 1e-5 of thr")
    assert flips <= max(10, int(near[-1].sum()))


def test_checkerboard_overflows_capacity_and_the_driver_retries():
    from unicorn_b200 import ops
    from unicorn_b200 import results as R
    from unicorn_b200.mots import MaskEncoder
    h, w = 720, 1280  # r = 1: the resized mask is the source itself
    cb = ((torch.arange(HIN)[:, None] + torch.arange(WIN)[None, :]) % 2).float()
    masks = torch.stack([cb, 1 - cb]).cuda()
    order, emit = torch.tensor([0, 1], dtype=torch.int32), [True, True]
    want, _ = reference(masks, order, emit, 1.0, h, w)
    need = len(want[0]) + len(want[1])
    cap, sentinel = 4096, 0xAB
    buf = torch.full((cap + 4096,), sentinel, dtype=torch.uint8, device="cuda")
    offsets = torch.zeros(3, dtype=torch.int64, device="cuda")
    ws = ops.mots_encode_workspace(2, h, w, "cuda")
    ops.mots_encode(masks, order.cuda(), torch.ones(2, dtype=torch.uint8, device="cuda"), THR, 1.0, h, w, ws, buf[:cap], offsets)
    torch.cuda.synchronize()
    assert offsets.tolist() == [0, len(want[0]), need]
    assert bytes(buf[:cap].cpu().numpy()) == (want[0] + want[1]).encode()[:cap]
    assert (buf[cap:] == sentinel).all()
    small, large = MaskEncoder(2, "cuda", capacity=64), MaskEncoder(2, "cuda", capacity=need + 1)
    assert run(small, masks, order, emit, 1.0, h, w) == run(large, masks, order, emit, 1.0, h, w) == want
    assert small.d_chars.numel() >= need
    assert R.rle_decode(want[0], h, w).sum() == h * w // 2


def test_captured_encode_equals_eager(blobs):
    from unicorn_b200 import ops
    h, w = 402, 640
    r = ratio(h, w)
    order, emit = order_and_emit(20, 64, 3)
    d_order, d_emit = order.cuda(), torch.tensor(emit, dtype=torch.uint8, device="cuda")
    ws = ops.mots_encode_workspace(20, h, w, "cuda")
    eager_c, eager_o = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda"), torch.zeros(21, dtype=torch.int64, device="cuda")
    ops.mots_encode(blobs, d_order, d_emit, THR, r, h, w, ws, eager_c, eager_o)
    chars, offs = torch.zeros_like(eager_c), torch.zeros_like(eager_o)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.mots_encode(blobs, d_order, d_emit, THR, r, h, w, ws, chars, offs)
    g.replay()
    torch.cuda.synchronize()
    n = int(eager_o[-1])
    assert n > 0 and torch.equal(offs, eager_o) and torch.equal(chars[:n], eager_c[:n])


# ---------------------------------------------------------------------------------------------------------------- driver
def _frames(n):
    from unicorn_b200.synthetic import make_video
    frames, _ = make_video(n, 320, 320, seed=1, n_obj=3)
    return frames


def _tracker(eng, use_graph):
    from unicorn_b200.mots import UnicornMOTSTracker
    from unicorn_b200.tracker import QuasiDenseEmbedTracker
    return UnicornMOTSTracker(eng, (320, 320), conf=0.01, nms=0.7, score_thr=0.02, max_dets=16, min_box_area=300, use_graph=use_graph,
                              tracker=QuasiDenseEmbedTracker(init_score_thr=0.05, obj_score_thr=0.03))


def test_pipelined_graph_driver_equals_sequential_and_host_path():
    from unicorn_b200 import results as R
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.weights import make_state_dict
    name, T = "unicorn_track_tiny_mask", 8
    eng = UnicornEngine(make_state_dict(name, 0), name)
    frames = _frames(T)
    sizes = [(201, 201), (480, 640)]  # 201 x 201 from a 320 x 320 input: 200 x 200 masks
    assert F.interpolate(torch.zeros(1, 1, 320, 320), scale_factor=1 / (320 / 201))[0, 0, :201, :201].shape == (200, 200)
    seq_trk, seq = _tracker(eng, False), []
    for t in range(T):
        h, w = sizes[t % 2]
        fr = seq_trk.step_tensor(frames[t:t + 1], h, w)
        last = seq_trk.last
        if last["rows"].numel():
            m = resized(last["masks"], last["rows"], min(320 / h, 320 / w), h, w) > seq_trk.mask_thres
        else:
            m = torch.zeros(0, h, w, dtype=torch.bool)
        want = R.mots_frame_result(t + 1, last["boxes"], last["ids"], m.cpu(), h, w, seq_trk.min_box_area)
        assert fr == want, t
        seq.append(fr)
    assert sum(len(f[1]) for f in seq) > 0, "no tracked instance"
    pipe_trk, pipe = _tracker(eng, True), []
    pipe_trk.submit(frames[0:1], *sizes[0])
    for t in range(1, T):
        pipe_trk.submit(frames[t:t + 1], *sizes[t % 2])
        pipe.append(pipe_trk.collect())
    pipe.append(pipe_trk.collect())
    assert all(s.graph is not None for s in pipe_trk._ctxs)
    assert pipe == seq


def test_mots_challenge_model_vs_oracle_and_one_driver_frame():
    import unicorn_oracle as orc
    from unicorn_b200 import ops
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.mots import UnicornMOTSTracker
    from unicorn_b200.weights import make_state_dict
    name = "unicorn_track_large_mot_challenge_mask"
    sd = make_state_dict(name, 0)
    img = _frames(1)[0:1]
    with torch.no_grad():
        (outs, locs, dyn, lvls, mf, um), _ = orc.whole_forward(img, sd, dict(orc.CONFIGS["unicorn_track_large_mot_challenge"], mask=True))
    eng = UnicornEngine(sd, name)
    eng.begin_frame()
    fpn, _ = eng.backbone(img.cuda(), tag="t")
    head = eng.head(fpn, None, "mot", with_masks=True)
    e_mf, e_um = eng.mask_branch(fpn)
    # tolerances of test_whole_gpu.py (bf16 operands against the fp32 oracle)
    rel = lambda a, b: ((a.float().cpu() - b).abs().max() / (b.abs().max() + 1e-12)).item()  # noqa: E731
    strides = torch.cat([torch.full((h * w,), float(s)) for (h, w), s in zip([(40, 40), (20, 20), (10, 10)], (8, 16, 32))])
    h = head.float().cpu()
    assert h.shape == outs.shape == (1, 2100, 6)
    assert ((h[0, :, :2] - outs[0, :, :2]).abs().max(dim=1)[0] / strides).max() < 0.2
    assert (torch.log(h[0, :, 2:4]) - torch.log(outs[0, :, 2:4])).abs().max() < 0.2
    assert (h[..., 4:] - outs[..., 4:]).abs().max() < 5e-2
    e_dyn = torch.cat([d[0, :, :, :169].reshape(-1, 169) for d in eng.dyn_levels], 0)
    assert rel(e_dyn[::16], dyn[0, ::16]) < 8e-2
    assert rel(e_mf.permute(0, 3, 1, 2), mf) < 8e-2 and rel(e_um.permute(0, 3, 1, 2)[0, :, ::4, ::4], um[0, :, ::4, ::4]) < 8e-2
    # NMS: the same decisions as the oracle on the same (oracle) head output
    ws = ops.PostWorkspace(2100, "cuda")
    d, cnt = ops.postprocess_device(outs[0].contiguous().cuda(), 1, 0.001, 0.7, ws)
    n = int(cnt.item())
    ref = orc.postprocess(outs.clone(), 1, 0.001, 0.7)[0]
    assert n == (0 if ref is None else ref.shape[0])
    if n:
        assert torch.cdist(d[:n, :6].cpu(), ref[:, :6], p=float("inf")).min(dim=0)[0].max().item() < 1e-4
    # dynamic masks of the engine's detections against the oracle's mask head on the engine's own head outputs
    d, cnt = ops.postprocess_device(head[0], 1, 0.001, 0.7, ws)
    n = min(int(cnt.item()), 4)
    if n:
        hw = [(t.shape[1], t.shape[2]) for t in eng.dyn_levels]
        masks = ops.dynamic_masks(e_mf, e_um, eng.dyn_levels, hw, ws, n, up_rate=4, d_rate=2)
        od, om = orc.postprocess_inst(head.cpu(), locs, e_dyn.cpu()[None], lvls, e_mf.permute(0, 3, 1, 2).cpu(),
                                      e_um.permute(0, 3, 1, 2).cpu(), 1, 0.001, 0.7, d_rate=2, max_masks=n)
        assert torch.allclose(od[:n], d[:n].cpu(), atol=1e-4)
        assert (om[:n, 0] - masks[:n].cpu()).abs().max() < 1e-3
    trk = UnicornMOTSTracker(eng, (320, 320), conf=0.001, score_thr=0.0, min_box_area=0)
    fr = trk.step_tensor(img, 402, 640)
    assert fr[0] == 1 and fr[2:5] == (2, 402, 640) and len(fr[1]) == len(fr[5])

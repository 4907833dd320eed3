"""ResNet-50 tracking models (unicorn_track_r50, unicorn_track_r50_mask) on the H100 path: the fused stem kernel, the residual-then-
activation conv epilogue, the 1x1 stride-2 downsample convs, the backbone against the CPU oracle, and the drivers end to end.

Tolerances: backbone outputs 4e-2 of the tensor's max (as for ConvNeXt, tests/test_engine_gpu.py); head as tests/test_engine_gpu.py."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).abs().max() / (b.abs().max() + 1e-12)).item()


def nchw(t):
    return t.float().permute(0, 3, 1, 2).cpu()


# ------------------------------------------------------------------------------------------------ uc_resnet_stem
@pytest.mark.parametrize("H,W", [(320, 320), (800, 1280), (328, 344)])  # 328 x 344: pooled 82 x 86, not a multiple of the 8 x 16 tile
@pytest.mark.parametrize("u8", [True, False])
def test_resnet_stem_vs_fp64(H, W, u8):
    """conv7x7s2 + folded BN + ReLU + maxpool3x3s2 against fp64 torch.  Error bound per output: the fp16 rounding of the folded
    weights (and of a non-integer fp32 input) contributes at most 2 * 2^-11 * sum|w||x| over the window, the bf16 output rounding
    2^-9 |y| (bounded here by 2^-8 |y|), plus 1e-3 for fp32 accumulation."""
    from unicorn_b200 import ops
    from unicorn_b200.weights import fold_bn
    g = torch.Generator().manual_seed(H * 7 + W + u8)
    w = torch.randn(64, 3, 7, 7, generator=g) / 147 ** 0.5
    sd = {"bn.weight": 1 + 0.1 * torch.randn(64, generator=g), "bn.bias": 0.1 * torch.randn(64, generator=g),
          "bn.running_mean": 10 * torch.randn(64, generator=g), "bn.running_var": 2e4 * (0.5 + torch.rand(64, generator=g))}
    wf, bf = fold_bn(w.double(), sd, "bn.")
    img = torch.randint(0, 256, (1, H, W, 3), generator=g, dtype=torch.uint8)
    x64 = img.permute(0, 3, 1, 2).double()
    if not u8:
        x64 = x64 + torch.rand(x64.shape, generator=g, dtype=torch.float64).float().double()  # non-integer fp32 pixels too
    ref = F.max_pool2d(F.relu(F.conv2d(x64, wf, bf, stride=2, padding=3)), 3, 2, 1)
    bound = F.max_pool2d(2 * 2.0 ** -11 * F.conv2d(x64.abs(), wf.abs(), stride=2, padding=3), 3, 2, 1) + 2.0 ** -8 * ref.abs() + 1e-3
    dev_in = img.cuda() if u8 else x64.float().contiguous().cuda()
    out = ops.resnet_stem(dev_in, ops.pack_resnet_stem_weight(wf.float().cuda()), bf.float().cuda())
    torch.cuda.synchronize()
    assert out.shape == (1, H // 4, W // 4, 64)
    err = (nchw(out).double() - ref).abs()
    assert (err <= bound).all(), (err.max().item(), (err - bound).max().item())


def test_resnet_stem_rejects_bad_shapes():
    from unicorn_b200 import ops
    from unicorn_b200._lib import UnicornB200Error
    w = torch.zeros(64, 160, dtype=torch.float16, device="cuda")
    b = torch.zeros(64, device="cuda")
    with pytest.raises(UnicornB200Error):
        ops.resnet_stem(torch.zeros(1, 3, 322, 320, device="cuda"), w, b, out=torch.empty(1, 80, 80, 64, dtype=torch.bfloat16, device="cuda"))


# ------------------------------------------------------------------------------------------------ uc_conv2d act_after_res
def _q(t):
    return t.to(torch.bfloat16).float()


def _conv_res_case(B, H, W, Cin, Cout, k, stride, block_n, out_slice=False):
    from unicorn_b200 import ops
    g = torch.Generator().manual_seed(B * 1000 + H * 31 + Cin + Cout + k + block_n)
    x = _q(torch.randn(B, H, W, Cin, generator=g))
    w = _q(torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5)
    bias = 0.1 * torch.randn(Cout, generator=g)
    pad = (k - 1) // 2
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    res = _q(torch.randn(B, Ho, Wo, Cout, generator=g))
    y = F.conv2d(x.permute(0, 3, 1, 2), w, bias, stride=stride, padding=pad).permute(0, 2, 3, 1) + res
    ref = F.relu(y)
    xd, resd = x.cuda().to(torch.bfloat16), res.cuda().to(torch.bfloat16)
    if out_slice:  # output into a channel slice of a wider buffer, residual read from the same slice (in place)
        big = torch.zeros(B, Ho, Wo, 2 * Cout, dtype=torch.bfloat16, device="cuda")
        out = big[..., Cout:]
        out.copy_(resd)
        resd = out
    else:
        out = torch.empty(B, Ho, Wo, Cout, dtype=torch.bfloat16, device="cuda")
    ops.conv2d(xd, ops.pack_conv_weight(w.cuda()), k, k, stride, pad, bias=bias.cuda(), act=1, res=resd, out=out, block_n=block_n,
               act_after_res=True)
    torch.cuda.synchronize()
    return out.float().cpu(), ref


@pytest.mark.parametrize("block_n", [0, 16, 32, 64, 96, 128, 192, 256, 1128, 1192, 1256])
def test_conv_act_after_res_block_n(block_n):
    """y = relu(conv + bias + res) for every N tile (1128/1192/1256: 2-CTA cluster variants); 1x1 with a partial M tile (1150 pixels)
    and 3x3 on an odd map."""
    for case in [(1, 1, 1150, 256, 512, 1, 1), (1, 13, 21, 64, 256, 3, 1)]:
        got, ref = _conv_res_case(*case, block_n=block_n)
        assert rel(got, ref) < 1e-2, (case, block_n, rel(got, ref))
        assert (got >= 0).all()


def test_conv_act_after_res_in_place_slice():
    got, ref = _conv_res_case(1, 20, 20, 128, 256, 1, 1, 0, out_slice=True)
    assert rel(got, ref) < 1e-2


@pytest.mark.parametrize("H,W,Cin,Cout", [(200, 320, 256, 512), (50, 80, 1024, 2048), (25, 41, 64, 128)])
def test_conv_1x1_stride2_vs_torch(H, W, Cin, Cout):
    """the downsample convs of ResNet-50 (1x1, stride 2, no padding) through conv_gemm's stride-phase maps, odd maps included."""
    from unicorn_b200 import ops
    g = torch.Generator().manual_seed(H + W + Cin)
    x = _q(torch.randn(1, H, W, Cin, generator=g))
    w = _q(torch.randn(Cout, Cin, 1, 1, generator=g) / Cin ** 0.5)
    b = 0.1 * torch.randn(Cout, generator=g)
    ref = F.conv2d(x.permute(0, 3, 1, 2), w, b, stride=2).permute(0, 2, 3, 1)
    got = ops.conv2d(x.cuda().to(torch.bfloat16), ops.pack_conv_weight(w.cuda()), 1, 1, 2, 0, bias=b.cuda())
    torch.cuda.synchronize()
    assert got.shape == ref.shape and rel(got, ref) < 1e-2


def test_conv_act_after_res_invalid_combinations():
    from unicorn_b200 import ops
    from unicorn_b200._lib import UnicornB200Error
    x = torch.zeros(1, 8, 8, 64, dtype=torch.bfloat16, device="cuda")
    w = torch.zeros(64, 1, 64, dtype=torch.bfloat16, device="cuda")
    res = torch.zeros_like(x)
    ones = torch.ones(64, device="cuda")
    bad = [dict(act=1),                                                                      # no residual
           dict(act=3, res=res), dict(act=0, res=res),                                       # ReLU only
           dict(act=1, res=res, gamma=ones),                                                 # layer scale
           dict(act=1, res=res, gn_stats=torch.zeros(1, 16, 2, dtype=torch.int64, device="cuda"), gn_groups=16)]
    for kw in bad:
        with pytest.raises(UnicornB200Error, match=r"code -1\)"):
            ops.conv2d(x, w, 1, 1, out=torch.empty_like(x), act_after_res=True, **kw)
    ops.conv2d(x, w, 1, 1, act=1, res=res, out=torch.empty_like(x), act_after_res=True)  # the valid form still launches


# ------------------------------------------------------------------------------------------------ backbone and frame vs the oracle
@pytest.mark.parametrize("H,W", [(320, 320), (800, 1280)])
def test_backbone_vs_oracle(H, W):
    import resnet_oracle as ro
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.weights import make_state_dict
    name = "unicorn_track_r50"
    sd = make_state_dict(name, 0)
    frames, _ = make_video(1, H, W, seed=3)
    with torch.no_grad():
        ref = ro.resnet50_features(frames[0:1], sd, ro.CONFIGS[name])
    eng = UnicornEngine(sd, name, autotune=False)
    eng.begin_frame()
    feats, seq = eng.features(frames[0:1].cuda().contiguous())
    torch.cuda.synchronize()
    errs = [rel(nchw(f), r) for f, r in zip(feats, ref)]
    print("R50 layer2/3/4 vs oracle", (H, W), errs)
    assert [tuple(nchw(f).shape) for f in feats] == [tuple(r.shape) for r in ref]
    assert max(errs) < 4e-2, errs
    assert seq["feat"].data_ptr() == feats[1].data_ptr() and seq["feat"].shape[-1] == 1024


@pytest.fixture(scope="module")
def sot_r50():
    import unicorn_oracle as orc
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.weights import make_state_dict
    name = "unicorn_track_r50"
    sd = make_state_dict(name, 0)
    frames, boxes = make_video(5, 320, 320, seed=0)
    return dict(name=name, sd=sd, frames=frames, boxes=boxes, eng=UnicornEngine(sd, name), orc=orc)


def test_sot_frame_vs_oracle(sot_r50):
    import resnet_oracle as ro
    from unicorn_b200.sot import UnicornSOTTrack
    s = sot_r50
    o = ro.SOTOracle(s["sd"], s["name"])
    o.initialize(s["frames"][0:1], s["boxes"][0, 0])
    st = {}
    o.track(s["frames"][2:3], st)
    trk = UnicornSOTTrack(s["eng"], (320, 320), use_graph=False, full_nms=True)
    trk.initialize_tensor(s["frames"][0:1], s["boxes"][0, 0])
    trk.track_tensor(s["frames"][2:3])
    torch.cuda.synchronize()
    last = trk.last
    errs = {f"fpn{i}": rel(nchw(last["fpn"][i]), st["fpn"][i]) for i in range(3)}
    errs["feat"] = rel(nchw(last["feat"]), st["feat"])
    errs["coarse"] = (last["priors"][0].cpu() - st["coarse"][0]).abs().max().item()
    head, href = last["head"].cpu(), st["head"]
    errs["score"] = (head[..., 4:] - href[..., 4:]).abs().max().item()
    print("R50 SOT frame vs oracle", errs)
    assert errs["feat"] < 4e-2 and max(errs[f"fpn{i}"] for i in range(3)) < 8e-2, errs
    assert errs["coarse"] < 6e-2 and errs["score"] < 5e-2, errs


def test_sot_three_in_flight_with_graphs_matches_sequential(sot_r50):
    from unicorn_b200.sot import UnicornSOTTrack
    s = sot_r50
    frames, box = s["frames"], s["boxes"][0, 0]
    seq = UnicornSOTTrack(s["eng"], (320, 320), use_graph=False)
    seq.initialize_tensor(frames[0:1], box)
    ref = [seq.track_tensor(frames[t:t + 1]) for t in range(1, 5)]
    pipe = UnicornSOTTrack(s["eng"], (320, 320), use_graph=True, depth=3)
    pipe.initialize_tensor(frames[0:1], box)
    got = []
    for t in range(1, 5):
        pipe.submit(frames[t:t + 1])
        if t >= 3:
            got.append(pipe.collect())
    while len(got) < 4:
        got.append(pipe.collect())
    for t, (r, g) in enumerate(zip(ref, got)):
        assert r[1] == g[1] and torch.equal(r[0], g[0]), f"frame {t + 1}: detections differ"


def test_mot_tracker_head_matches_compat_whole_mode():
    from unicorn_b200.compat.model import UnicornB200Model
    from unicorn_b200.mot import UnicornMOTTracker
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.tracker import QuasiDenseEmbedTracker
    from unicorn_b200.weights import make_state_dict
    name = "unicorn_track_r50"
    sd = make_state_dict(name, 0)
    model = UnicornB200Model(sd, name)
    frames, _ = make_video(3, 320, 320, seed=1, n_obj=3)
    mot = UnicornMOTTracker(model.engine, (320, 320), conf=0.01, nms=0.7, score_thr=0.02,
                            tracker=QuasiDenseEmbedTracker(init_score_thr=0.05, obj_score_thr=0.03))
    for t in range(3):
        boxes, ids = mot.step_tensor(frames[t:t + 1].cuda())
        head = mot.last["head"].clone()
        whole, seq = model(imgs=frames[t:t + 1].cuda(), mode="whole")
        torch.cuda.synchronize()
        assert torch.equal(head, whole), f"frame {t}: MOT head differs from whole mode"
        assert seq["feat"].shape == (1, 1024, 20, 20)
    assert mot.last["dets"].shape[0] > 0


def test_mask_model_whole_mode_and_vos_run():
    """unicorn_track_r50_mask: whole mode returns UnicornHeadMask's tuple with the R50 widths; mask branch refines read 512/1024/2048."""
    import resnet_oracle as ro
    from unicorn_b200.compat.model import UnicornB200Model
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.weights import make_state_dict
    name = "unicorn_track_r50_mask"
    sd = make_state_dict(name, 0)
    model = UnicornB200Model(sd, name)
    frames, _ = make_video(1, 320, 320, seed=1, n_obj=3)
    (out, locs, dyn, lvls, mf, um), _ = model(imgs=frames[0:1].cuda(), mode="whole")
    with torch.no_grad():
        (o_out, _, o_dyn, _, o_mf, o_um), _ = ro.whole_forward(frames[0:1], sd, ro.CONFIGS[name])
    torch.cuda.synchronize()
    assert (out.cpu()[..., 4:] - o_out[..., 4:]).abs().max().item() < 5e-2
    assert rel(dyn, o_dyn) < 8e-2 and rel(mf, o_mf) < 8e-2 and rel(um, o_um) < 8e-2


# ------------------------------------------------------------------------------------------------ reference goldens
def test_r50_mask_whole_mode_vs_reference_golden():
    """unicorn_track_r50_mask `mode="whole"` head and detections against tests/golden/whole_r50_mask_320.npz with the criteria of
    tests/test_whole_gpu.py (check_head / check_dets)."""
    import numpy as np
    import unicorn_oracle as orc
    from unicorn_b200.compat.model import UnicornB200Model, postprocess
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.weights import make_state_dict
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from test_whole_gpu import check_dets, check_head
    g = np.load(os.path.join(ROOT, "tests", "golden", "whole_r50_mask_320.npz"))
    name = str(g["config"])
    frames, _ = make_video(2, 320, 320, seed=int(g["seed_video"]), n_obj=int(g["n_obj"]))
    img = frames[int(g["frame"]):int(g["frame"]) + 1].cuda()
    model = UnicornB200Model(make_state_dict(name, 0), name)
    (out, locs, dyn, lvls, mf, um), seq = model(imgs=img, mode="whole")
    check_head(out, g["head"])
    assert rel(dyn[0, ::16], torch.from_numpy(g["dyn_sub"])) < 8e-2 and rel(mf, torch.from_numpy(g["mask_feats"])) < 8e-2
    assert rel(seq["feat"][0, ::8], torch.from_numpy(g["feat_sub"])) < 4e-2
    dets = postprocess(out.clone(), 8, float(g["conf"]), float(g["nms"]))[0].cpu()
    check_dets(dets, g["dets"], orc)


def test_r50_sot_box_vs_reference_golden(sot_r50):
    """UnicornSOTTrack on unicorn_track_r50 (frame 2 of the golden sequence): the head within the check_head criteria and the tracked
    box (top-1 detection) on the reference's box."""
    import numpy as np
    from unicorn_b200.sot import UnicornSOTTrack
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from test_whole_gpu import check_head
    g = np.load(os.path.join(ROOT, "tests", "golden", "sot_r50_320.npz"))
    from unicorn_b200.synthetic import make_video
    s = sot_r50
    nf = int(g["n_frames"])
    frames, boxes = make_video(nf, 320, 320, seed=int(g["seed"]))
    trk = UnicornSOTTrack(s["eng"], (320, 320), use_graph=False, full_nms=True)
    trk.initialize_tensor(frames[0:1], boxes[0, 0])
    dets, n = trk.track_tensor(frames[nf - 1:nf])
    check_head(trk.last["head"], g["head"])
    ref = g["dets"]
    iou = s["orc"].box_iou_np(dets[:1, :4].numpy(), ref[:1, :4])[0, 0]
    assert n > 0 and iou > 0.7, (iou, dets[:1], ref[:1])
    assert rel(nchw(trk.last["feat"])[0, ::8], torch.from_numpy(g["feat_sub"])) < 4e-2

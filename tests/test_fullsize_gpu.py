"""BASELINE.json's full sizes (ConvNeXt-L, 800x1280, N = 16000 correlation positions): size-independent properties of the
kernels plus one full frame against the CPU oracle (2-3 s of oracle time per frame on the GPU box's host cores)."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
dev = "cuda"
torch.backends.cudnn.allow_tf32 = False          # the torch references below must be true fp32
torch.backends.cuda.matmul.allow_tf32 = False


def G(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def test_corr_full_size_properties():
    """N = 16000 x 16000 (the similarity matrix would be 512 MB in fp16): columns of the softmax sum to one, the operator
    is linear in V, and 192 sampled current positions match an fp32 evaluation of exactly those columns."""
    from unicorn_b200 import ops
    g = G(1)
    N, C = 16000, 128
    k = (torch.randn(N, C, generator=g) * 0.5).to(dev).half()
    q = (torch.randn(N, C, generator=g) * 0.5).to(dev).half()
    ones = torch.ones(1, N, device=dev)
    out = ops.corr_propagate(k, q, ones)
    assert (out - 1).abs().max().item() < 2e-3          # sum_i softmax(S)[i, j] == 1
    v = torch.rand(3, N, generator=g).to(dev)
    o3 = ops.corr_propagate(k, q, v)
    comb = ops.corr_propagate(k, q, (v[0] + 2 * v[1] - 0.5 * v[2])[None].contiguous())
    assert (comb[0] - (o3[0] + 2 * o3[1] - 0.5 * o3[2])).abs().max().item() < 2e-3   # linearity in V
    cols = torch.randperm(N, generator=g)[:192].to(dev)
    S = k.float() @ q.float()[cols].t()                  # [N, 192] fp32: only the sampled columns
    ref = v @ torch.softmax(S, dim=0)
    assert (o3[:, cols] - ref).abs().max().item() < 2e-3
    assert torch.equal(o3, ops.corr_propagate(k, q, v))  # deterministic


@pytest.mark.parametrize("M_hw,Cin,Cout,k,extra", [((50, 80), 768, 3072, 1, "gelu"), ((50, 80), 3072, 768, 1, "res"), ((25, 40), 1536, 6144, 1, "gelu"),
                                                  ((100, 160), 256, 256, 3, "gn"), ((200, 320), 192, 768, 1, "gelu"), ((100, 160), 384, 768, 2, "")])
def test_conv_full_layer_shapes(M_hw, Cin, Cout, k, extra):
    """uc_conv2d on ConvNeXt-L@800x1280 layer shapes (whatever N tile the heuristic picks) against an fp32 evaluation of 256
    sampled output pixels on the same bf16-rounded operands."""
    from unicorn_b200 import ops
    g = G(2)
    H, W = M_hw
    s = 2 if k == 2 else 1
    pad = 1 if k == 3 else 0
    x = torch.randn(1, H, W, Cin, generator=g).to(dev).bfloat16()
    w = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).to(dev)
    bias = torch.randn(Cout, generator=g).to(dev)
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    res = torch.randn(1, Ho, Wo, Cout, generator=g).to(dev).bfloat16() if extra == "res" else None
    gamma = torch.randn(Cout, generator=g).to(dev) if extra == "res" else None
    st = torch.zeros(1, 16, 2, device=dev, dtype=torch.int64) if extra == "gn" else None
    out = ops.conv2d(x, ops.pack_conv_weight(w), k, k, s, pad, bias=bias, act=ops.ACT_GELU if extra == "gelu" else 0, gamma=gamma, res=res,
                     gn_stats=st, gn_groups=16 if extra == "gn" else 0)
    wq = w.bfloat16().float()
    full = F.conv2d(x.float().permute(0, 3, 1, 2), wq, bias, stride=s, padding=pad) if Cin * Cout * k * k <= 256 * 256 * 9 else None
    idx = torch.randperm(Ho * Wo, generator=g)[:256]
    xf = F.unfold(x.float().permute(0, 3, 1, 2), k, padding=pad, stride=s)[0][:, idx.to(dev)]     # [Cin*k*k, 256]
    ref = (wq.reshape(Cout, -1) @ xf).t() + bias                                                    # [256, Cout]
    if extra == "gelu":
        ref = F.gelu(ref)
    if extra == "res":
        ref = ref * gamma + res.float().reshape(-1, Cout)[idx.to(dev)]
    got = out.float().reshape(-1, Cout)[idx.to(dev)]
    err = (got - ref).abs().max().item() / (ref.abs().max().item() + 1e-9)
    assert err < 6e-3, err
    if st is not None:  # GroupNorm statistics of the full map (fixed-point 2^22) against the fp32 map
        y = full[0].reshape(16, -1)
        ssum = st[0, :, 0].double() / 4194304.0
        ssq = st[0, :, 1].double() / 4194304.0
        assert torch.allclose(ssum, y.double().sum(1), rtol=1e-3, atol=2.0)
        assert torch.allclose(ssq, (y.double() ** 2).sum(1), rtol=1e-3)


def test_large_frame_vs_oracle_and_determinism():
    """One ConvNeXt-L 800x1280 SOT frame: engine vs the CPU oracle (fp32) stage by stage, and two engine runs bit-identical."""
    import unicorn_oracle as orc
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.sot import UnicornSOTTrack
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.weights import make_state_dict
    name = "unicorn_track_large"
    sd = make_state_dict(name, 0)
    frames, boxes = make_video(2, 800, 1280, seed=0)
    eng = UnicornEngine(sd, name)
    trk = UnicornSOTTrack(eng, (800, 1280), use_graph=False, full_nms=True)
    trk.initialize_tensor(frames[0:1], boxes[0, 0])
    dets, n = trk.track_tensor(frames[1:2])
    head1 = trk.last["head"].clone()
    prior1 = trk.last["priors"][0].clone()
    dets2, n2 = trk.track_tensor(frames[1:2])
    assert n2 == n and torch.equal(dets2, dets) and torch.equal(trk.last["head"], head1)      # deterministic
    assert head1.shape == (1, 21000, 6) and torch.isfinite(head1).all()
    assert (head1[..., 4:] >= 0).all() and (head1[..., 4:] <= 1).all()
    from bench import host_threads
    nthr = torch.get_num_threads()
    torch.set_num_threads(host_threads())  # the box shows 128 CPUs behind a 16-CPU cgroup quota
    try:
        o = orc.SOTOracle(sd, name)
        o.initialize(frames[0:1], boxes[0, 0])
        st = {}
        o.track(frames[1:2], st)
    finally:
        torch.set_num_threads(nthr)
    rel = lambda a, b: ((a.float().cpu() - b).abs().max() / (b.abs().max() + 1e-12)).item()  # noqa: E731
    nchw = lambda t: t.float().permute(0, 3, 1, 2)  # noqa: E731
    errs = {"feat": rel(nchw(trk.last["feat"]), st["feat"]), "embed_cur": rel(nchw(trk.last["embed_cur"]), st["embed_cur"]),
            "fpn0": rel(nchw(trk.last["fpn"][0]), st["fpn"][0]), "fpn2": rel(nchw(trk.last["fpn"][2]), st["fpn"][2]),
            "coarse": (prior1.cpu() - st["coarse"][0]).abs().max().item(),
            "head_score": (head1.cpu()[..., 4:] - st["head"][..., 4:]).abs().max().item()}
    print("large-frame errors:", {k: f"{v:.3e}" for k, v in errs.items()})
    # same tolerances as the tiny model (test_engine_gpu.py)
    tol = dict(feat=4e-2, embed_cur=5e-2, fpn0=8e-2, fpn2=8e-2, coarse=6e-2, head_score=5e-2)
    bad = {k: v for k, v in errs.items() if not v <= tol[k]}
    assert not bad, f"out of tolerance: {bad} (all: {errs})"


def _with_host_threads(fn):
    from bench import host_threads
    nthr = torch.get_num_threads()
    torch.set_num_threads(host_threads())  # the box shows 128 CPUs behind a 16-CPU cgroup quota
    try:
        with torch.no_grad():
            return fn()
    finally:
        torch.set_num_threads(nthr)


def test_mot_frame_1536x2048_vs_oracle():
    """BASELINE configs[2]: one ConvNeXt-L 1536x2048 frame in `mode="whole"` (conv M = 49 152 pixels at stride 8, 64 512 anchors,
    8 classes) + the QDTrack embedding branch, engine vs the CPU oracle (fp32); ~5.9 TFLOP of oracle work."""
    import tracker_oracle as to
    import unicorn_oracle as orc
    from unicorn_b200 import ops
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.mot import UnicornMOTTracker
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.weights import make_state_dict
    name, H, W = "unicorn_track_large", 1536, 2048
    sd = make_state_dict(name, 0)
    frames, _ = make_video(1, H, W, seed=2, n_obj=6)
    eng = UnicornEngine(sd, name)
    trk = UnicornMOTTracker(eng, (H, W), conf=0.01, nms=0.7)
    trk.submit(frames[0:1])
    torch.cuda.synchronize()
    head = trk.last["head"].clone()
    emb = trk.last["embed"].float().permute(0, 3, 1, 2).cpu()
    n = int(trk.ws.count.item())
    dets = trk.ws.dets[:n].cpu()
    feats = trk.feats[:min(n, trk.max_dets)].cpu()
    trk.collect()
    assert head.shape == (1, 64512, 13) and torch.isfinite(head).all()
    cfg = orc.CONFIGS[name]

    def oracle():
        o_head, seq = orc.whole_forward(frames[0:1], sd, cfg)
        _, f_cur = orc.deform_interaction(seq, seq, sd)  # frame 1: pre_dict = cur_dict (mot_evaluator.py:1014-1015)
        return o_head, orc.upsample_embed(f_cur, sd)
    o_head, o_emb = _with_host_threads(oracle)
    stride = torch.cat([torch.full((m,), float(s)) for m, s in ((192 * 256, 8), (96 * 128, 16), (48 * 64, 32))])
    h = head.cpu()
    errs = dict(xy=((h[0, :, :2] - o_head[0, :, :2]).abs().max(dim=1)[0] / stride).max().item(),
                logwh=(torch.log(h[0, :, 2:4]) - torch.log(o_head[0, :, 2:4])).abs().max().item(),
                score=(h[..., 4:] - o_head[..., 4:]).abs().max().item(),
                embed=((emb - o_emb).abs().max() / o_emb.abs().max()).item())
    print("1536x2048 MOT frame errors vs oracle:", {k: f"{v:.3e}" for k, v in errs.items()})
    assert errs["xy"] < 0.2 and errs["logwh"] < 0.2 and errs["score"] < 5e-2 and errs["embed"] < 5e-2, errs
    o_dets = orc.postprocess(o_head, 8, 0.01, 0.7)[0]
    assert o_dets is not None and abs(n - o_dets.shape[0]) <= max(5, 0.05 * o_dets.shape[0]), (n, o_dets.shape)
    # embedding sampling at the engine's own boxes against grid_sample on the engine's own map (a14, fp16 map)
    k = min(n, 64)
    ref_f = to.sample_embeddings(emb, dets[:k, :4], (H, W))
    assert (feats[:k] - ref_f).abs().max().item() < 2e-3 * max(1.0, ref_f.abs().max().item())


def test_vos_large_mask_3_objects_vs_oracle():
    """BASELINE configs[3]: unicorn_track_large_mask at 800x1280 with three objects — propagated priors, per-object mask-head scores,
    best-instance masks and the aggregated label map against the CPU oracle's VOS driver (fp32)."""
    import unicorn_oracle as orc
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.vos import UnicornVOSTrack
    from unicorn_b200.weights import make_state_dict
    name, H, W = "unicorn_track_large_mask", 800, 1280
    sd = make_state_dict(name, 0)
    frames, boxes = make_video(2, H, W, seed=4, n_obj=3)
    init = {str(i + 1): boxes[0, i] for i in range(3)}
    vos = UnicornVOSTrack(UnicornEngine(sd, name), (H, W))
    vos.debug = True
    vos.initialize_tensor(frames[0:1], init)
    out = vos.track_tensor(frames[1:2])
    seg = out["segmentation"].cpu().numpy()

    def oracle():
        o = orc.VOSOracle(sd, name)
        o.initialize(frames[0:1], init)
        return o.track(frames[1:2])
    o_seg, o_res = _with_host_threads(oracle)
    report = {}
    for oid in init:
        det, mask = out["objects"][oid]
        r = o_res[oid]
        assert det is not None and r["det"] is not None
        po = vos.last["per_obj"][oid]
        report[oid] = dict(coarse=(vos.last["coarse"][oid].cpu() - r["coarse"][0]).abs().max().item(),
                           score=(po["head"].cpu()[..., 4:] - r["head"][..., 4:]).abs().max().item(),
                           top1_iou=float(orc.box_iou_np(det[None, :4].numpy(), r["det"][None, :4].numpy())[0, 0]))
        mb, rb = mask.cpu() > 0.5, r["mask"] > 0.5
        report[oid]["mask_iou"] = float((mb & rb).sum() / max(1, (mb | rb).sum()))
        assert report[oid]["coarse"] < 6e-2 and report[oid]["score"] < 5e-2, report
    agree = float((seg == o_seg).mean())
    import numpy as np
    o_soft = np.stack([np.asarray(o_res[o]["soft"], dtype=np.float32) for o in init])
    chans = np.concatenate([np.prod(1 - o_soft, axis=0, keepdims=True), o_soft], 0)
    top2 = np.sort(chans, axis=0)[-2:]
    cond = (top2[1] - top2[0]) > 0.25  # pixels whose label is a well-conditioned argmax (seeded random weights: noise-like soft masks)
    agree_cond = float((seg == o_seg)[cond].mean()) if cond.any() else 1.0
    print("large-mask VOS, 3 objects:", report, "label agreement", agree, "where the oracle's margin > 0.25:", agree_cond, "fraction", float(cond.mean()))
    assert agree_cond > 0.99
    out_dir = os.environ.get("UC_REPORT_DIR", "")  # optional directory for the measured parity reports
    if os.path.isdir(out_dir):
        import json
        json.dump(dict(per_object=report, label_agreement=agree, label_agreement_margin_0p25=agree_cond, margin_fraction=float(cond.mean())), open(os.path.join(out_dir, "r2_vos_large_parity.json"), "w"), indent=1)
    # where the engine picks the oracle's instance its mask must be the oracle's mask (bf16 features: IoU, not bit equality)
    for oid, rr in report.items():
        if rr["top1_iou"] > 0.9:
            assert rr["mask_iou"] > 0.9, report

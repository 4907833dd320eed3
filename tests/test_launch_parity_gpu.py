"""Every kernel launch of full-size production frames against an fp32 reference of that launch.

The unit tests check each kernel at shapes, strides and N tiles their authors picked; the frame tests compare whole frames with the CPU
oracle at tolerances that absorb ~500 bf16 layers.  Here the leaf launchers of unicorn_b200.ops (the functions that call _lib.check)
are wrapped while the drivers run real frames eagerly, and every launch is held to its unit test's tolerance at the shape, view, N
tile and epilogue variant production uses:

  value      a reference of the launch (fp32, float64 where the unit test uses it) computed from snapshots of its operands taken just
             before it, so in-place launches are checked against what they overwrote;
  footprint  every byte of every argument's storage outside the launch's declared output elements, and every buffer the engine owns
             (activations, GroupNorm / LayerNorm statistics arenas, work counters), is bitwise unchanged by the launch: a column
             written past a channel slice of a concat buffer lands in the sibling slice, not in a guard column;
  coverage   every uc_* entry point that reaches _lib.check inside a checked frame went through a checked launcher (counts equal per
             entry point), and the entry points the frame is expected to reach did appear.

Launches inside CUDA-graph capture (the plan-time autotuner times candidate N tiles in graphs) pass through unchecked and uncounted;
the summary lists the layers tuned at plan time, since those ran a tile no committed table chose.  The wrapper synchronises the
device around every launch, so the streams are serialised: cross-stream races are the subject of the graph-vs-eager and
pipelined-vs-sequential bit-identity tests, not of this file."""
import contextlib
import ctypes
import functools
import inspect
import json
import os
import sys
import time
from collections import Counter, defaultdict

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

FIX = float(1 << 22)  # fixed-point scale of the GroupNorm / LayerNorm statistics the kernels accumulate
ACTS = {0: lambda t: t, 1: F.relu, 2: F.gelu, 3: F.silu, 4: torch.sigmoid}


# ------------------------------------------------------------------------------------------------ storage helpers (CPU and GPU)
def storage_key(t):
    return (t.device, t.untyped_storage().data_ptr())


def storage_bytes(t):
    """Flat uint8 view of the whole storage under the view t."""
    return torch.empty(0, dtype=torch.uint8, device=t.device).set_(t.untyped_storage())


def output_mask(nbytes, views, device="cpu"):
    """bool [nbytes]: True on every byte of the elements of `views` (tensors, or (dtype, size, stride, storage_offset) tuples, all in
    one storage of nbytes bytes)."""
    m = torch.zeros(nbytes, dtype=torch.bool, device=device)
    for v in views:
        dt, size, stride, off = (v.dtype, tuple(v.shape), v.stride(), v.storage_offset()) if torch.is_tensor(v) else v
        es = torch.empty(0, dtype=dt).element_size()
        e = torch.zeros(nbytes // es, dtype=torch.bool, device=device)
        e.as_strided(size, stride, off).fill_(True)
        m[:e.numel() * es] |= e[:, None].expand(-1, es).reshape(-1)
    return m


class Snapshot:
    """Copies of the whole storages under a set of tensors, taken before a launch."""

    def __init__(self, tensors):
        self.st = {}
        for t in tensors:
            if t is None or not t.is_cuda or t.untyped_storage().nbytes() == 0:
                continue
            k = storage_key(t)
            if k not in self.st:
                live = storage_bytes(t)
                self.st[k] = (live, live.clone())

    def pre(self, t):
        """t as it was before the launch (t itself if its storage was not snapshotted: allocated by the launcher)."""
        if t is None or not torch.is_tensor(t):
            return t
        s = self.st.get(storage_key(t)) if t.is_cuda else None
        if s is None:
            return t
        return s[1].view(t.dtype).as_strided(t.shape, t.stride(), t.storage_offset())

    def changed_outside(self, outs):
        """[(storage nbytes, first changed byte outside `outs`, count)] over the snapshotted storages."""
        per = defaultdict(list)
        for o in outs:
            if o is not None and o.numel():
                per[storage_key(o)].append(o)
        bad = []
        for k, (live, old) in self.st.items():
            diff = live != old
            if k in per:
                diff &= ~output_mask(live.numel(), per[k], live.device)
            n = int(diff.sum())
            if n:
                bad.append((live.numel(), int(diff.nonzero()[0, 0]), n))
        return bad


def _tensors(v):
    from unicorn_b200 import ops
    if torch.is_tensor(v):
        yield v
    elif isinstance(v, (list, tuple)):
        for x in v:
            yield from _tensors(x)
    elif isinstance(v, ops.PostWorkspace):
        yield from (v.buf, v.dets, v.count, v.anchors)


def _desc(t):
    return None if t is None else [list(t.shape), list(t.stride()), str(t.dtype).replace("torch.", "")]


# ------------------------------------------------------------------------------------------------ comparisons (err / tol)
def ratio(got, ref, rel, abs_=1e-6):
    """max|got - ref| / (rel * max|ref| + abs_): the unit tests' close()."""
    if ref.numel() == 0:
        return 0.0
    got, ref = got.double(), ref.double()
    return (got - ref).abs().max().item() / (rel * ref.abs().max().item() + abs_)


def elem_ratio(got, ref, atol, rtol=0.0):
    """max over elements of |got - ref| / (atol + rtol * |ref|): allclose-style bounds."""
    if ref.numel() == 0:
        return 0.0
    got, ref = got.double(), ref.double()
    return ((got - ref).abs() / (atol + rtol * ref.abs())).max().item()


def exact(got, ref):
    return 0.0 if got.shape == ref.shape and torch.equal(got, ref.to(got.dtype)) else float("inf")


def nchw(t):
    return t.permute(0, 3, 1, 2)


class Checked:
    """What a launch's check returns: err / tol per output, the declared output views, variant tags and a description."""

    def __init__(self, ratios, outs, tags=(), **info):
        self.ratios, self.outs, self.tags, self.info = ratios, outs, list(tags), info


# ------------------------------------------------------------------------------------------------ references of the launchers
def c_conv2d(a, ret, pre):
    """test_conv_epilogue_gpu: F.conv2d on the launch's rounded operands, LN fold from row_stats, bias / act / gamma / residual (or
    relu(pre + res)), GroupNorm statistics of the pre-activation in float64."""
    x, wp, KH, KW = pre(a["x"]), pre(a["w_packed"]), a["KH"], a["KW"]
    Cout, Cin = wp.shape[0], x.shape[3]
    pre_act = F.conv2d(nchw(x.float()), wp.float().reshape(Cout, KH, KW, Cin).permute(0, 3, 1, 2), None, stride=a["stride"],
                       padding=a["pad"])
    B, _, H, W = pre_act.shape
    tags = [f"bn{a['block_n']}", {0: "none", 1: "relu", 2: "gelu", 3: "silu", 4: "sigmoid"}[a["act"]]]
    if a["row_stats"] is not None:  # LayerNorm folded in: y = rstd (W'x) - rstd mu colsum(W') + c
        rs = pre(a["row_stats"]).double().reshape(-1, 2) / FIX
        mu = rs[:, 0] / Cin
        rstd = 1.0 / torch.sqrt((rs[:, 1] / Cin - mu * mu).clamp(min=0) + a["row_eps"])
        r = rstd.float().view(B, H, W, 1).permute(0, 3, 1, 2)
        m = mu.float().view(B, H, W, 1).permute(0, 3, 1, 2)
        pre_act = r * pre_act - (r * m) * pre(a["col_s"])[:Cout].float().view(1, -1, 1, 1)
        tags.append("row_stats")
    if a["bias"] is not None:
        pre_act = pre_act + pre(a["bias"])[:Cout].view(1, -1, 1, 1)
    res = nchw(pre(a["res"]).float()) if a["res"] is not None else None
    if res is not None:
        tags.append("res_inplace" if storage_key(a["res"]) == storage_key(ret) else "res")
    if a["act_after_res"]:
        ref = F.relu(pre_act + res)
        tags.append("act_after_res")
    else:
        ref = ACTS[a["act"]](pre_act)
        if a["gamma"] is not None:
            ref = ref * pre(a["gamma"])[:Cout].view(1, -1, 1, 1)
            tags.append("gamma")
        if res is not None:
            ref = ref + res
    if ret.dtype == torch.float32:
        tags.append("f32out")
    if ret.stride(2) != ret.shape[3]:
        tags.append("slice_out")
    ratios = {"y": ratio(ret, ref.permute(0, 2, 3, 1), 1e-4 if ret.dtype == torch.float32 else 4e-3, 1e-3)}
    outs = [ret]
    if a["gn_stats"] is not None:
        G = a["gn_groups"]
        got = (a["gn_stats"].reshape(B, G, 2) - pre(a["gn_stats"]).reshape(B, G, 2)).double() / FIX
        pg = pre_act.double().reshape(B, G, Cout // G, -1)
        want = torch.stack([pg.sum(dim=(2, 3)), (pg * pg).sum(dim=(2, 3))], -1)
        ratios["gn_stats"] = elem_ratio(got, want, 2.0, 1e-3)
        outs.append(a["gn_stats"])
        tags.append(f"gn{G}")
    return Checked(ratios, outs, tags, x=_desc(a["x"]), y=_desc(ret), k=KH, s=a["stride"], block_n=a["block_n"])


def c_groupnorm_apply(a, ret, pre):
    """test_conv_gn_silu_prior: scale / shift from the statistics snapshot in float64 (as the kernel), act, + prior * beta; the second
    output + add2."""
    x = pre(a["x"]).float()
    B, H, W, C = x.shape
    G = a["G"]
    st = pre(a["stats"]).double().reshape(B, G, 2) / FIX
    n = H * W * (C // G)
    mean = st[..., 0] / n
    rstd = 1.0 / torch.sqrt((st[..., 1] / n - mean * mean).clamp(min=0) + a["eps"])
    scale = rstd.repeat_interleave(C // G, 1) * pre(a["w"]).double()
    shift = pre(a["b"]).double() - mean.repeat_interleave(C // G, 1) * scale
    y = ACTS[a["act"]]((x * scale.float()[:, None, None] + shift.float()[:, None, None]))
    tags = []
    if a["prior"] is not None:
        y = y + pre(a["prior"]).float().reshape(B, H, W, 1) * pre(a["beta"]).float().view(1, 1, 1, C)
        tags.append("prior")
    ratios = {"y": ratio(ret, y, 1e-2)}
    outs = [ret]
    if a["out2"] is not None:
        ratios["y2"] = ratio(a["out2"], y + pre(a["add2"]).float(), 1.2e-2)
        outs.append(a["out2"])
        tags.append("out2")
    if a["out"] is None:
        tags.append("inplace")
    return Checked(ratios, outs, tags, x=_desc(a["x"]), G=G)


def dw_taps_from_qtab(q, C):
    """The bf16 taps [C,1,7,7] and fp32 biases [C] that uc_dwconv7_mma's operand (ops.pack_dw_weight_mma) carries: per 32-channel
    chunk [32][7][8] tap pairs {e[j-1], e[j]} (e[-1] = 0), then 32 biases."""
    nch = q.shape[0]
    lo = q[:, :1792].reshape(nch, 32, 7, 8)[..., 1:8] & 0xFFFF  # tap k = e[k], the low half of pair k + 1
    taps = ((lo ^ 0x8000) - 0x8000).to(torch.int16).view(torch.bfloat16).float()
    bias = q[:, 1792:].contiguous().view(torch.float32).reshape(-1)
    return taps.reshape(nch * 32, 1, 7, 7)[:C].contiguous(), bias[:C].contiguous()


def c_dwconv7_mma(a, ret, pre):
    x = pre(a["x"]).float()
    C = x.shape[3]
    w, b = dw_taps_from_qtab(pre(a["qtab"]), C)
    ref = F.conv2d(nchw(x), w, b, padding=3, groups=C).permute(0, 2, 3, 1)
    return Checked({"y": ratio(ret, ref, 5e-3)}, [ret, a["work_counter"]], x=_desc(a["x"]))


def c_dwconv7(a, ret, pre):
    x = pre(a["x"]).float()
    C = x.shape[3]
    w = pre(a["w49"]).t().reshape(C, 1, 7, 7)
    ref = F.conv2d(nchw(x), w, pre(a["bias"]), padding=3, groups=C).permute(0, 2, 3, 1)
    ratios, outs, tags = {"y": ratio(ret, ref, 5e-3)}, [ret, a["work_counter"]], []
    if a["ln_stats"] is not None:  # sum / sum of squares over C of the STORED outputs
        of = ret.double().reshape(-1, C)
        got = (a["ln_stats"] - pre(a["ln_stats"])).double().reshape(-1, 2) / FIX
        ratios["ln_stats"] = elem_ratio(got, torch.stack([of.sum(1), (of * of).sum(1)], 1), 1e-3, 1e-5)
        outs.append(a["ln_stats"])
        tags.append("ln_stats")
    return Checked(ratios, outs, tags, x=_desc(a["x"]))


def c_convnext_mlp(a, ret, pre):
    """test_convnext_mlp_fused: LN -> bf16 -> w1f, + c1 -> GELU -> bf16 -> w2, + b2 -> * gamma -> + x."""
    t = pre(a["t"]).float()
    M, C = t.shape
    tn = F.layer_norm(t, (C,), None, None, a["eps"]).bfloat16().float()
    hid = F.gelu(tn @ pre(a["w1f"]).float().reshape(4 * C, C).t() + pre(a["c1"])).bfloat16().float()
    ref = pre(a["x"]).float() + pre(a["gamma"]) * (hid @ pre(a["w2"]).float().reshape(C, 4 * C).t() + pre(a["b2"]))
    return Checked({"x": ratio(a["x"], ref, 6e-3)}, [a["x"]], x=_desc(a["x"]))


def c_layernorm(a, ret, pre):
    x = pre(a["x2d"]).float()
    if a["res"] is not None:
        x = x + pre(a["res"]).float()
    ref = F.layer_norm(x, (x.shape[1],), pre(a["w"]), pre(a["b"]), a["eps"])
    tags = ["inplace"] if a["out"] is not None and storage_key(a["out"]) == storage_key(a["x2d"]) else []
    if ret.stride(0) != ret.shape[1]:
        tags.append("rows_view")
    return Checked({"y": ratio(ret, ref, 6e-3)}, [ret], tags, x=_desc(a["x2d"]), y=_desc(ret))


def c_stem_ln(a, ret, pre):
    img = pre(a["img"])
    u8 = img.dtype == torch.uint8
    x = nchw(img.float()) if u8 else img
    C0 = a["w48"].shape[1]
    y = F.conv2d(x, pre(a["w48"]).t().reshape(C0, 3, 4, 4), pre(a["bias"]), stride=4).permute(0, 2, 3, 1)
    ref = F.layer_norm(y, (C0,), pre(a["lnw"]), pre(a["lnb"]), a["eps"])
    return Checked({"y": ratio(ret, ref, 6e-3)}, [ret], ["u8"] if u8 else [], img=_desc(a["img"]))


def c_resnet_stem(a, ret, pre):
    """test_resnet_stem_vs_fp64: float64 conv7x7 s2 + bias + ReLU + maxpool on the launch's fp16 weights, that test's bound."""
    img = pre(a["img"])
    u8 = img.dtype == torch.uint8
    x64 = nchw(img).double() if u8 else img.double()
    w = pre(a["w160"])[:, :147].double().reshape(64, 3, 7, 7)
    ref = F.max_pool2d(F.relu(F.conv2d(x64, w, pre(a["bias"]).double(), stride=2, padding=3)), 3, 2, 1)
    bound = F.max_pool2d(2 * 2.0 ** -11 * F.conv2d(x64.abs(), w.abs(), stride=2, padding=3), 3, 2, 1) + 2.0 ** -8 * ref.abs() + 1e-3
    r = ((nchw(ret).double() - ref).abs() / bound).max().item()
    return Checked({"y": r}, [ret], ["u8"] if u8 else [], img=_desc(a["img"]))


def c_copy_upsample(a, ret, pre):
    up = a["up"]
    ref = pre(a["src"]).repeat_interleave(up, 1).repeat_interleave(up, 2)
    return Checked({"y": exact(a["dst"], ref)}, [a["dst"]], dst=_desc(a["dst"]))


def c_pixel_shuffle2(a, ret, pre):
    ref = F.pixel_shuffle(nchw(pre(a["x"]).float()), 2).permute(0, 2, 3, 1)
    return Checked({"y": exact(ret, ref)}, [ret], y=_desc(ret))


def c_bilinear(a, ret, pre):
    src = pre(a["src"])
    Hs, Ws = src.shape[-2:]
    s = src.reshape(1, -1, Hs, Ws)
    if a["scale_h"] > 0:
        ref = F.interpolate(s, scale_factor=(1.0 / a["scale_h"], 1.0 / a["scale_w"]), mode="bilinear", align_corners=False)
    else:
        ref = F.interpolate(s, size=(a["Hd"], a["Wd"]), mode="bilinear", align_corners=False)
    assert ref.shape[-2:] == (a["Hd"], a["Wd"])
    return Checked({"y": ratio(ret.reshape(ref.shape), ref, 1e-6)}, [ret], src=_desc(a["src"]), Hd=a["Hd"], Wd=a["Wd"])


def c_head_decode(a, ret, pre):
    rows = []
    for (h, w), s, r, c in zip(a["hw"], a["strides"], a["regobj"], a["cls"]):
        r, c = pre(r).reshape(h * w, -1), pre(c).reshape(h * w, -1)
        yv, xv = torch.meshgrid(torch.arange(h, device=r.device), torch.arange(w, device=r.device), indexing="ij")
        grid = torch.stack((xv, yv), 2).view(-1, 2).float()
        rows.append(torch.cat([(r[:, :2] + grid) * s, torch.exp(r[:, 2:4]) * s, torch.sigmoid(r[:, 4:5]),
                               torch.sigmoid(c[:, :a["ncls"]])], 1))
    return Checked({"y": ratio(ret[0], torch.cat(rows, 0), 1e-6)}, [ret], hw=a["hw"], ncls=a["ncls"])


def c_letterbox_u8(a, ret, pre):
    import preprocess_oracle as po
    ref, r = po.letterbox(pre(a["src"]).cpu().numpy(), tuple(a["input_size"]), swap_rb=a["swap_rb"], pad=a["pad"])
    out, r2 = ret
    return Checked({"y": exact(out[0].cpu(), torch.from_numpy(ref)), "r": 0.0 if r == r2 else float("inf")}, [out],
                   src=_desc(a["src"]), size=list(a["input_size"]))


def c_nchw_to_nhwc(a, ret, pre):
    return Checked({"y": exact(ret, pre(a["x"]).permute(0, 2, 3, 1).to(ret.dtype))}, [ret], x=_desc(a["x"]))


def c_copy_rows_if(a, ret, pre):
    take = (int(pre(a["flag"])[0]) != 0) != bool(a["invert"])
    ref = pre(a["src"]) if take else pre(a["dst"])
    return Checked({"y": exact(a["dst"], ref)}, [a["dst"]], ["copied" if take else "kept"], dst=_desc(a["dst"]))


def msda_reference(value, offlog, level_hw, M, P):
    """test_msda_random_and_fused: grid-point reference points, offsets / logits from offlog, softmax over L*P, grid_sample (bilinear,
    zeros, align_corners False) per level (ms_deform_attn_core_pytorch)."""
    S, D, L = value.shape[0], 32, len(level_hw)
    off = offlog[:, :M * L * P * 2].reshape(S, M, L, P, 2)
    attn = torch.softmax(offlog[:, M * L * P * 2:M * L * P * 3].reshape(S, M, L * P), -1).reshape(S, M, L, P)
    refs = []
    for (h, w) in level_hw:
        ry, rx = torch.meshgrid(torch.linspace(0.5, h - 0.5, h), torch.linspace(0.5, w - 0.5, w), indexing="ij")
        refs.append(torch.stack((rx.reshape(-1) / w, ry.reshape(-1) / h), -1))
    ref_pts = torch.cat(refs, 0).to(value.device)
    norm = torch.tensor([[w, h] for (h, w) in level_hw], dtype=torch.float32, device=value.device)
    loc = ref_pts[:, None, None, None, :] + off / norm[None, None, :, None, :]  # (S, M, L, P, 2)
    vals = value.view(S, M, D).split([h * w for h, w in level_hw], dim=0)
    out = torch.zeros(M, D, S, device=value.device)
    for lid, (h, w) in enumerate(level_hw):
        v = vals[lid].permute(1, 2, 0).reshape(M, D, h, w)
        grid = (2 * loc[:, :, lid] - 1).permute(1, 0, 2, 3)  # (M, S, P, 2)
        smp = F.grid_sample(v, grid, mode="bilinear", padding_mode="zeros", align_corners=False)  # (M, D, S, P)
        out += (smp * attn[:, :, lid].permute(1, 0, 2)[:, None]).sum(-1)
    return out.permute(2, 0, 1).reshape(S, M * D)


def c_msda_fused(a, ret, pre):
    ref = msda_reference(pre(a["value"]).float(), pre(a["offlog"]).float(), a["level_hw"], a["M"], a["P"])
    return Checked({"y": ratio(ret, ref, 6e-3)}, [ret], value=_desc(a["value"]), offlog=_desc(a["offlog"]), hw=a["level_hw"])


def c_corr_propagate(a, ret, pre):
    """V @ softmax(K Q^T, dim=0), in chunks of current positions (16 000^2 fp32 does not fit as one matrix)."""
    K, Q, V = pre(a["embed_ref"]).float(), pre(a["embed_cur"]).float(), pre(a["values"]).float()
    ref = torch.empty(V.shape[0], Q.shape[0], device=V.device)
    for c0 in range(0, Q.shape[0], 2048):
        ref[:, c0:c0 + 2048] = V @ torch.softmax(K @ Q[c0:c0 + 2048].t(), dim=0)
    return Checked({"y": ratio(ret, ref, 2e-4)}, [ret], [f"rows{V.shape[0]}"], n_ref=K.shape[0], n_cur=Q.shape[0],
                   values=_desc(a["values"]))


def c_postprocess_device(a, ret, pre):
    """oracle.postprocess (pinned to the reference) on the same pred; with max_keep, the first max_keep rows of the full result.  The
    kept anchors must decode to the kept boxes (the mask head reads its parameters through them)."""
    import unicorn_oracle as orc
    ws, pred = a["ws"], pre(a["pred"])
    ref = orc.postprocess(pred.cpu()[None].clone(), a["ncls"], a["conf"], a["nms"])[0]
    n_ref = 0 if ref is None else ref.shape[0]
    want = min(a["max_keep"], n_ref) if a["max_keep"] else n_ref
    n = int(ws.count[0])
    ratios = {"count": 0.0 if n == want else float("inf")}
    if want and n == want:
        got = ws.dets[:n].cpu()
        ratios["rows"] = elem_ratio(got, ref[:n], 1e-5)
        p = pred[ws.anchors[:n].long()].cpu()
        box = torch.cat([p[:, :2] - p[:, 2:4] / 2, p[:, :2] + p[:, 2:4] / 2], 1)
        ratios["anchors"] = elem_ratio(box, got[:, :4], 1e-5)
    return Checked(ratios, [ws.buf, ws.dets, ws.count, ws.anchors], [f"max_keep{a['max_keep']}"], A=pred.shape[0], ncls=a["ncls"],
                   kept=n)


def c_sample_embed(a, ret, pre):
    import tracker_oracle as to
    emb = nchw(pre(a["embed"]).float())
    h, w = emb.shape[2:]
    s = a["stride"]
    k = a["n_max"] if a["count"] is None else min(int(pre(a["count"])[0]), a["n_max"])
    ref = to.sample_embeddings(emb, pre(a["boxes"])[:k, :4].float(), (h * s, w * s), s=s) if k else ret[:0]
    return Checked({"y": elem_ratio(ret[:k], ref.reshape(k, -1), 2e-3, 1e-5)}, [ret], n=k, embed=_desc(a["embed"]))


def c_bisoftmax(a, ret, pre):
    f = pre(a["det_embeds"]).float() @ pre(a["memo_embeds"]).float().t()
    ref = (f.softmax(1) + f.softmax(0)) / 2
    if a["det_labels"] is not None:
        ref = ref * (pre(a["det_labels"])[:, None] == pre(a["memo_labels"])[None, :]).float()
    return Checked({"y": elem_ratio(ret, ref, 1e-5, 1e-4)}, [ret], N=f.shape[0], M=f.shape[1])


def c_box_iou(a, ret, pre):
    import tracker_oracle as to
    assert not a["plus_one"], "the +1 convention (ByteTrack) has no reference here"
    ref = to.box_iou(pre(a["a"]).float(), pre(a["b"]).float())
    return Checked({"y": elem_ratio(ret, ref, 1e-6, 1e-5)}, [ret], N=ref.shape[0], M=ref.shape[1])


def c_qd_assign(a, ret, pre):
    """The reference loop of test_qd_assign_kernel_matches_reference_loop (quasi_dense_embed_tracker.py:188-199)."""
    s2, memo, box = pre(a["scores"]).cpu().clone(), pre(a["memo_ids"]).cpu(), pre(a["boxes5"]).cpu()
    N = s2.shape[0]
    ref = torch.full((N,), -1, dtype=torch.long)
    for i in range(N):
        conf, j = torch.max(s2[i], dim=0)
        if conf > a["match_thr"] and memo[j] > -1:
            if box[i, 4] > a["obj_thr"]:
                ref[i] = memo[j]
                s2[:i, j] = 0
                s2[i + 1:, j] = 0
            elif conf > a["nms_conf_thr"]:
                ref[i] = -2
    return Checked({"ids": exact(ret.cpu(), ref)}, [ret], N=N, M=s2.shape[1])


def c_aligned_bilinear_add(a, ret, pre):
    """oracle.aligned_bilinear + the snapshot of dst; bound: one bf16 rounding of the result, 2^-8 |ref| (+1e-6)."""
    import unicorn_oracle as orc
    ref = pre(a["dst"]).float() + orc.aligned_bilinear(nchw(pre(a["src"]).float()), a["factor"]).permute(0, 2, 3, 1)
    r = ((a["dst"].double() - ref.double()).abs() / (2.0 ** -8 * ref.double().abs() + 1e-6)).max().item()
    return Checked({"y": r}, [a["dst"]], [f"x{a['factor']}"], src=_desc(a["src"]), dst=_desc(a["dst"]))


def c_dynamic_masks(a, ret, pre):
    """Per kept anchor (ws.anchors[:count]): its 169 controller outputs, relative coordinates, the three 1x1 layers, convex upsampling,
    sigmoid (oracle.dynamic_masks), aligned x d_rate (oracle.aligned_bilinear) — fp32 on the CPU.  Only rows < count are outputs."""
    import unicorn_oracle as orc
    ws = a["ws"]
    n = min(int(pre(ws.count)[0]), a["n_max"])
    mf, um = nchw(pre(a["mask_feats"]).cpu()).contiguous(), nchw(pre(a["up_masks"]).cpu()).contiguous()
    anchors = pre(ws.anchors)[:n].cpu().long()
    starts = np.cumsum([0] + [h * w for h, w in a["level_hw"]])
    worst = 0.0
    for c0 in range(0, n, 8):
        prm, loc, lvl = [], [], []
        for an in anchors[c0:c0 + 8].tolist():
            k = int(np.searchsorted(starts, an, side="right") - 1)
            ai, wk = an - starts[k], a["level_hw"][k][1]
            d = pre(a["dyn_levels"][k])
            prm.append(d.reshape(-1, d.shape[-1])[ai, :169].cpu())
            loc.append(torch.tensor([(ai % wk + 0.5) * a["strides"][k], (ai // wk + 0.5) * a["strides"][k]]))
            lvl.append(k)
        m = orc.dynamic_masks(mf, torch.stack(prm), torch.stack(loc), torch.tensor(lvl), um, up_rate=a["up_rate"], soi=tuple(a["soi"]))
        ref = orc.aligned_bilinear(m, a["d_rate"])[:, 0]
        worst = max(worst, elem_ratio(ret[c0:c0 + len(prm)].cpu(), ref, 1e-4))
    return Checked({"masks": worst}, [ret[:n], a["scratch"]], [f"n_max{a['n_max']}"], n=n, out=_desc(ret))


def c_mots_encode(a, ret, pre):
    """The host path of test_mots_encode_gpu (F.interpolate + threshold + results.overlap_free + results.rle_encode).  Strings must
    be byte-identical, except that a resized value within 1e-5 of the threshold may round to either side (in the instance itself or
    in an earlier one, which hides the pixel): those pixels, and only those, may differ, as in that file's smooth-mask test."""
    from unicorn_b200 import results as R
    order, emit = pre(a["order"]).long(), pre(a["emit"]).bool().tolist()
    k, H, W, thr, chars = order.numel(), a["H"], a["W"], a["thr"], a["chars"]
    offs = a["offsets"][:k + 1].cpu().tolist()
    if k == 0:
        return Checked({"strings": 0.0 if offs == [0] else float("inf")}, [a["ws"], a["chars"], a["offsets"][:1]], k=0)
    v = F.interpolate(pre(a["masks"])[order][:, None], scale_factor=1 / a["r"], mode="bilinear", align_corners=False)[:, 0, :H, :W]
    free = R.overlap_free(v > thr).cpu().numpy()
    want = [R.rle_encode(free[i]) if emit[i] else "" for i in range(k)]
    want_offs = np.cumsum([0] + [len(s) for s in want]).tolist()
    cap = chars.numel()  # the driver grows the buffer and encodes again when offsets[k] exceeds it: only the prefix is written
    text = bytes(chars[:min(offs[k], cap)].cpu().numpy()).decode("ascii")
    if offs == want_offs and text == "".join(want)[:cap]:
        ratios = {"strings": 0.0}
    elif offs[k] > cap:
        ratios = {"strings": float("inf")}
    else:
        got = [text[offs[i]:offs[i + 1]] for i in range(k)]
        near = (((v - thr).abs() < 1e-5).cumsum(0) > 0).cpu()
        bad = flips = 0
        for i in range(k):
            if got[i] == want[i]:
                continue
            if not emit[i]:
                bad += 1
                continue
            diff = torch.from_numpy(R.rle_decode(got[i], H, W) ^ R.rle_decode(want[i], H, W))
            bad += int((diff & ~near[i]).sum())
            flips += int(diff.sum())
        ratios = {"strings": float("inf") if bad else 0.0, "flips": flips / max(10.0, float(near[-1].sum()))}
    return Checked(ratios, [a["ws"], a["chars"], a["offsets"][:k + 1]], k=k, H=H, W=W, chars=offs[k], capacity=cap)


def c_vos_aggregate(a, ret, pre):
    """test_vos_aggregate_kernel_matches_definition: soft masks resized by 1/r into a zero map (init label maps as 0 / 1), float32
    background product in list order, argmax with the lower channel winning ties; the label map must be exact wherever the
    decision is not a tie within the soft masks' own tolerance (2e-6)."""
    ids, H0, W0 = a["ids"], a["seg"].shape[0], a["seg"].shape[1]
    soft_ref = torch.zeros(len(ids), H0, W0, device=a["seg"].device)
    for k, oid in enumerate(ids):
        if k < len(a["masks"]):
            m = F.interpolate(pre(a["masks"][k]).reshape(1, 1, a["Hin"], a["Win"]), scale_factor=1 / a["r"], mode="bilinear",
                              align_corners=False)[0, 0, :H0, :W0]
            soft_ref[k, :m.shape[0], :m.shape[1]] = m
        else:
            soft_ref[k] = (pre(a["init_mask"]) == int(oid)).float()
    merge = torch.zeros(max(int(i) for i in ids) + 1, H0, W0, device=soft_ref.device)
    for k, oid in enumerate(ids):
        merge[int(oid)] = soft_ref[k]
    bg = torch.ones(H0, W0, device=soft_ref.device)
    for k in range(len(ids)):
        bg = bg * (1 - soft_ref[k])
    merge[0] = bg
    top2 = merge.topk(2, dim=0).values if merge.shape[0] > 1 else None
    clear = (top2[0] - top2[1]) > 4e-6 if top2 is not None else torch.ones_like(bg, dtype=torch.bool)
    seg_ref = merge.argmax(0).to(torch.uint8)
    ratios = {"soft": elem_ratio(a["soft"][:len(ids)], soft_ref, 2e-6),
              "seg": 0.0 if torch.equal(a["seg"][clear], seg_ref[clear]) else float("inf")}
    return Checked(ratios, [a["soft"][:len(ids)], a["seg"]], n=len(ids), H0=H0, W0=W0)


CHECKS = {name[2:]: fn for name, fn in globals().items() if name.startswith("c_")}
# launchers no production frame reaches: a call inside a checked frame fails until a reference is added here
NO_REFERENCE = ("dwconv7_ln", "add", "nhwc_to_nchw", "msda_forward")


def leaf_launchers():
    """The functions of unicorn_b200.ops that launch through _lib.check."""
    from unicorn_b200 import ops
    return sorted(n for n, f in vars(ops).items() if inspect.isfunction(f) and f.__module__ == ops.__name__ and "_lib.check(" in inspect.getsource(f))


# ------------------------------------------------------------------------------------------------ the harness
class LaunchMismatch(AssertionError):
    def __init__(self, kind, index, msg):
        super().__init__(f"{kind} check failed at checked launch #{index}: {msg}")
        self.kind, self.index = kind, index


class Harness:
    def __init__(self, monkeypatch):
        from unicorn_b200 import _lib, ops
        self.records, self.engines, self.seen = [], [], set()
        self.calls, self.checked = Counter(), Counter()
        self.depth, self.active, self.tamper, self.tuned = 0, False, None, []
        self.wall = time.time()
        monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)  # the references are true fp32
        monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
        leaves = leaf_launchers()
        assert set(leaves) == set(CHECKS) | set(NO_REFERENCE), ("launchers without a reference in this file",
                                                                sorted(set(leaves) ^ (set(CHECKS) | set(NO_REFERENCE))))
        orig_check = _lib.check

        def check(rc, what="", n=1):
            if self.active and not torch.cuda.is_current_stream_capturing():
                self.calls[what] += 1
                if self.depth:
                    self.checked[what] += 1
                    self._entry = what
            return orig_check(rc, what, n)
        monkeypatch.setattr(_lib, "check", check)
        for name in leaves:
            monkeypatch.setattr(ops, name, self._wrap(name, getattr(ops, name)))

    def engine(self, eng):
        self.engines.append(eng)
        return eng

    def _owned(self):
        for e in self.engines:
            yield from e._bufs.values()
            yield from (t for t in (e._stats_arena, e._row_arena, e._ctr_arena) if t is not None)

    def _wrap(self, name, fn):
        sig = inspect.signature(fn)
        check = CHECKS.get(name)

        @functools.wraps(fn)
        def launcher(*args, **kw):
            if not self.active or torch.cuda.is_current_stream_capturing():
                return fn(*args, **kw)
            assert check is not None, f"ops.{name} has no reference in this file"
            ba = sig.bind(*args, **kw)
            ba.apply_defaults()
            a = dict(ba.arguments)
            torch.cuda.synchronize()
            snap = Snapshot(list(_tensors(list(a.values()))) + list(self._owned()))
            self.depth += 1
            self._entry = None
            try:
                ret = fn(*args, **kw)
            finally:
                self.depth -= 1
            torch.cuda.synchronize()
            index = len(self.records)
            if self.tamper is not None:
                self.tamper(name, a, ret, index)
                torch.cuda.synchronize()
            if self._entry is None:  # returned without launching (an empty problem)
                return ret
            res = check(a, ret, snap.pre)
            rec = dict(op=name, entry=self._entry, tags=res.tags, ratios={k: float(v) for k, v in res.ratios.items()}, **res.info)
            rec["worst"] = max(rec["ratios"].values()) if rec["ratios"] else 0.0
            if not rec["worst"] <= 1.0:
                raise LaunchMismatch("value", index, json.dumps(rec, default=str))
            bad = snap.changed_outside(res.outs)
            if bad:
                raise LaunchMismatch("footprint", index, f"{rec['entry']} wrote outside its declared outputs: (storage bytes, first "
                                                         f"byte, bytes changed) {bad}; launch {json.dumps(rec, default=str)}")
            self.records.append(rec)
            self.seen.add(rec["entry"])
            self.seen.update(rec["entry"] + "+" + t for t in rec["tags"])
            return ret
        return launcher

    @contextlib.contextmanager
    def frame(self):
        """A checked region: at its end every counted launch must have gone through a checked launcher, per entry point."""
        tuned0 = [set(e._bn_cache) for e in self.engines]
        self.calls.clear()
        self.checked.clear()
        self.active = True
        try:
            yield
        finally:
            self.active = False
        for e, keys in zip(self.engines, tuned0):
            self.tuned += sorted(set(e._bn_cache) - keys)
        if self.calls != self.checked:
            unchecked = {k: self.calls[k] - self.checked[k] for k in self.calls if self.calls[k] != self.checked[k]}
            raise LaunchMismatch("coverage", len(self.records), f"launches that bypassed the checked launchers: {unchecked}")

    def finish(self, label, expected):
        """Per-op summary (printed, and written to $UC_REPORT_DIR); every expected entry point / variant must have been checked."""
        per = defaultdict(lambda: dict(launches=0, worst=0.0, worst_launch=None))
        for r in self.records:
            p = per[r["entry"]]
            p["launches"] += 1
            if r["worst"] >= p["worst"]:
                p["worst"], p["worst_launch"] = r["worst"], r
        bns = Counter(r.get("block_n") for r in self.records if r["entry"] == "uc_conv2d")
        report = dict(frame=label, wall_s=round(time.time() - self.wall, 1), launches=len(self.records), tuned_at_plan_time=self.tuned,
                      conv_block_n=dict(sorted((str(k), v) for k, v in bns.items())), per_op=dict(sorted(per.items())),
                      device=torch.cuda.get_device_name())
        print(f"\n[{label}] {len(self.records)} launches checked in {report['wall_s']} s on {report['device']}; conv N tiles {report['conv_block_n']}")
        for k, p in report["per_op"].items():
            print(f"  {k:28s} {p['launches']:5d} launches  worst err/tol {p['worst']:.3f}")
        if self.tuned:
            print("  tuned at plan time (not in the committed tables):", self.tuned)
        out_dir = os.environ.get("UC_REPORT_DIR", "")
        if os.path.isdir(out_dir):
            with open(os.path.join(out_dir, f"launch_parity_{label}.json"), "w") as f:
                json.dump(report, f, indent=1, default=str)
        missing = sorted(set(expected) - self.seen)
        assert not missing, f"expected entry points / variants not reached: {missing}"
        return report


@pytest.fixture
def harness(monkeypatch):
    h = Harness(monkeypatch)
    yield h
    h.engines.clear()
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ the production frames
BASE = {"uc_conv2d", "uc_groupnorm_apply", "uc_copy_upsample", "uc_dwconv7_mma", "uc_convnext_mlp", "uc_head_decode", "uc_postprocess",
        "uc_conv2d+slice_out", "uc_conv2d+res_inplace", "uc_conv2d+f32out", "uc_groupnorm_apply+inplace"}
CONVNEXT = {"uc_stem_ln", "uc_layernorm", "uc_layernorm+rows_view", "uc_layernorm+inplace"}
INTERACTION = {"uc_msda_fused_bf16", "uc_pixel_shuffle2", "uc_groupnorm_apply+out2"}
SOT = INTERACTION | {"uc_corr_propagate", "uc_bilinear_f32", "uc_groupnorm_apply+prior"}


def _engine(h, name, **kw):
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.weights import make_state_dict
    return h.engine(UnicornEngine(make_state_dict(name, 0), name, **kw))


def _bgr_u8(frames):
    """make_video frames (fp32 BGR NCHW) -> uint8 BGR HWC numpy images."""
    return frames.round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("ln_fold", [False, True], ids=["default", "ln_fold"])
def test_sot_large_800x1280_device_preproc(harness, ln_fold):
    """unicorn_track_large SOT: initialize + track on raw 1080x1920 RGB frames letterboxed on the device to 800x1280, full NMS."""
    from unicorn_b200.sot import UnicornSOTTrack
    from unicorn_b200.synthetic import make_video
    eng = _engine(harness, "unicorn_track_large", ln_fold=ln_fold)
    frames, boxes = make_video(2, 1080, 1920, seed=0)
    rgb = _bgr_u8(frames)[..., ::-1].copy()
    x1, y1, x2, y2 = boxes[0, 0].tolist()
    trk = UnicornSOTTrack(eng, (800, 1280), use_graph=False, full_nms=True, device_preproc=True)
    with harness.frame():
        trk.initialize(rgb[0], {"init_bbox": [x1, y1, x2 - x1, y2 - y1]})
    with harness.frame():
        trk.track(rgb[1])
    want = BASE | CONVNEXT | SOT | {"uc_letterbox_u8", "uc_stem_ln+u8"}
    if ln_fold:
        want |= {"uc_dwconv7+ln_stats", "uc_conv2d+row_stats"}
    harness.finish("sot_large" + ("_ln_fold" if ln_fold else ""), want)


@pytest.mark.gpu
def test_sot_r50_800x1280(harness):
    from unicorn_b200.sot import UnicornSOTTrack
    from unicorn_b200.synthetic import make_video
    eng = _engine(harness, "unicorn_track_r50")
    frames, boxes = make_video(2, 800, 1280, seed=1)
    trk = UnicornSOTTrack(eng, (800, 1280), use_graph=False, full_nms=True)
    with harness.frame():
        trk.initialize_tensor(frames[0:1], boxes[0, 0])
    with harness.frame():
        trk.track_tensor(frames[1:2])
    harness.finish("sot_r50", BASE | SOT | {"uc_resnet_stem", "uc_conv2d+act_after_res", "uc_layernorm"})


@pytest.mark.gpu
def test_mot_challenge_1536x2048_qd(harness):
    """unicorn_track_large_mot_challenge, QuasiDense arm, two 1536x2048 frames (49 152 pixels at stride 8, 64 512 anchors).  Seeded
    random weights give low scores: the score and new-tracklet gates are lowered to zero (as test_tracker_gpu lowers them) so that every
    detection of the first frame starts a tracklet and the second frame's association runs the bi-softmax and the assignment."""
    from unicorn_b200.mot import UnicornMOTTracker
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.tracker import QuasiDenseEmbedTracker
    eng = _engine(harness, "unicorn_track_large_mot_challenge")
    frames, _ = make_video(2, 1536, 2048, seed=2, n_obj=6)
    mot = UnicornMOTTracker(eng, (1536, 2048), conf=0.01, nms=0.7, score_thr=0.0,
                            tracker=QuasiDenseEmbedTracker(init_score_thr=0.0, obj_score_thr=0.03))
    for t in range(2):
        with harness.frame():
            mot.step_tensor(frames[t:t + 1])
    harness.finish("mot_1536x2048", BASE | CONVNEXT | INTERACTION | {"uc_copy_rows_if", "uc_sample_embed", "uc_box_iou", "uc_bisoftmax",
                                                                     "uc_qd_assign"})


@pytest.mark.gpu
def test_vos_large_mask_800x1280_3_objects(harness):
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.vos import UnicornVOSTrack
    eng = _engine(harness, "unicorn_track_large_mask")
    frames, boxes = make_video(2, 800, 1280, seed=4, n_obj=3)
    vos = UnicornVOSTrack(eng, (800, 1280))
    with harness.frame():
        vos.initialize_tensor(frames[0:1], {str(i + 1): boxes[0, i] for i in range(3)})
    with harness.frame():
        vos.track_tensor(frames[1:2])
    harness.finish("vos_large_mask", BASE | CONVNEXT | SOT | {"uc_aligned_bilinear_add", "uc_dynamic_masks", "uc_corr_propagate+rows3",
                                                              "uc_vos_aggregate", "uc_postprocess+max_keep1"})


@pytest.mark.gpu
def test_mots_challenge_mask_800x1280_from_1080x1920(harness):
    """unicorn_track_large_mot_challenge_mask MOTS: two 1080x1920 frames letterboxed to 800x1280 (uint8), the tracker's gates lowered so
    that the tracked instances' masks are encoded (uc_mots_encode with k > 0, at the original resolution)."""
    import preprocess_oracle as po
    from unicorn_b200.mots import UnicornMOTSTracker
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.tracker import QuasiDenseEmbedTracker
    eng = _engine(harness, "unicorn_track_large_mot_challenge_mask")
    frames, _ = make_video(2, 1080, 1920, seed=5, n_obj=4)
    raw = _bgr_u8(frames)
    trk = UnicornMOTSTracker(eng, (800, 1280), conf=0.01, nms=0.7, score_thr=0.0, max_dets=64, min_box_area=0,
                             tracker=QuasiDenseEmbedTracker(init_score_thr=0.0, obj_score_thr=0.0))
    ks = []
    for t in range(2):
        lb, _ = po.letterbox(raw[t], (800, 1280), swap_rb=False)
        with harness.frame():
            fr = trk.step_tensor(torch.from_numpy(lb)[None], 1080, 1920)
        ks.append(len(fr[5]))
    assert sum(ks) > 0, "no instance was encoded"
    harness.finish("mots_large_mask", BASE | CONVNEXT | INTERACTION | {"uc_dynamic_masks+n_max64", "uc_mots_encode", "uc_aligned_bilinear_add",
                                                                       "uc_copy_rows_if", "uc_sample_embed", "uc_stem_ln+u8"})


# ------------------------------------------------------------------------------------------------ the harness is not vacuous
def _tiny_frame(h):
    from unicorn_b200.synthetic import make_video
    eng = _engine(h, "unicorn_track_tiny")
    frames, _ = make_video(1, 320, 320, seed=0)
    img = frames.cuda()

    def run():
        eng.begin_frame()
        eng.backbone(img, tag="t")
    return eng, run


@pytest.mark.gpu
def test_tiny_frame_passes_the_harness(harness):
    """The controls below fail for the reason they inject, not because the tiny frame fails on its own."""
    _, run = _tiny_frame(harness)
    with harness.frame():
        run()
    harness.finish("tiny_control", {"uc_conv2d+slice_out", "uc_groupnorm_apply", "uc_convnext_mlp"})


@pytest.mark.gpu
def test_control_value_one_channel_off_by_one_percent(harness):
    _, run = _tiny_frame(harness)
    hit = []

    def tamper(name, a, ret, index):
        if name == "conv2d" and not hit and ret.dtype == torch.bfloat16 and ret.float().abs().max().item() > 2.0:
            # the channel holding max|y|: 1 % of it, after bf16 rounding, exceeds 4e-3 max|y| + 1e-3
            c = int(ret.float().abs().amax(dim=(0, 1, 2)).argmax())
            ret[..., c] *= 1.01
            hit.append(index)
    harness.tamper = tamper
    with pytest.raises(LaunchMismatch) as ei:
        with harness.frame():
            run()
    assert hit and ei.value.kind == "value" and ei.value.index == hit[0], (hit, str(ei.value))


@pytest.mark.gpu
def test_control_footprint_one_column_past_a_concat_slice(harness):
    _, run = _tiny_frame(harness)
    hit = []

    def tamper(name, a, ret, index):
        if name == "conv2d" and not hit and ret.dtype == torch.bfloat16 and ret.stride(2) > ret.shape[3]:
            # the element one column past the slice in pixel 0: the sibling slice of the concat buffer
            ret.view(torch.int16).as_strided((1,), (1,), ret.storage_offset() + ret.shape[3]).bitwise_xor_(1)
            hit.append(index)
    harness.tamper = tamper
    with pytest.raises(LaunchMismatch) as ei:
        with harness.frame():
            run()
    assert hit and ei.value.kind == "footprint" and ei.value.index == hit[0], (hit, str(ei.value))


@pytest.mark.gpu
def test_control_coverage_launch_around_the_launchers(harness):
    from unicorn_b200 import _lib, ops
    _, run = _tiny_frame(harness)
    a = torch.ones(4, 8, dtype=torch.bfloat16, device="cuda")
    out = torch.empty_like(a)
    with pytest.raises(LaunchMismatch) as ei:
        with harness.frame():
            run()
            _lib.check(_lib.lib().uc_add(ops._p(a), 8, ops._p(a), 8, ops._p(out), 8, ctypes.c_long(4), 8, ops.BF16, _lib.stream_ptr()), "uc_add")
    assert ei.value.kind == "coverage" and "uc_add" in str(ei.value), str(ei.value)
    assert torch.equal(out, a + a)


# ------------------------------------------------------------------------------------------------ CPU: the output-element mask
def test_output_mask_views():
    buf = torch.zeros(2, 3, 4, 10)  # [B, H, W, 10]: a concat buffer of a 6- and a 4-channel slice
    lo, hi = buf[..., :6], buf[..., 6:]
    nb = buf.untyped_storage().nbytes()
    m = output_mask(nb, [hi]).view(-1, 4).all(1).view(buf.shape)  # per element: all 4 bytes
    assert m[..., 6:].all() and not m[..., :6].any()
    assert torch.equal(output_mask(nb, [lo, hi]), torch.ones(nb, dtype=torch.bool))
    # rows view of a channel slice (engine._rows): [H*W, C] with the buffer's pixel stride
    s = buf[:1, ..., 2:6]
    rows = s.as_strided((3 * 4, 4), (s.stride(2), 1), s.storage_offset())
    m = output_mask(nb, [rows]).view(-1, 4).all(1).view(buf.shape)
    want = torch.zeros(buf.shape, dtype=torch.bool)
    want[0, ..., 2:6] = True
    assert torch.equal(m, want)
    # an in-place alias declares the same elements; a 2-D linear view ([M, C] as [1, 1, M, C])
    x = torch.zeros(12, 8, dtype=torch.bfloat16)
    x4 = x.as_strided((1, 1, 12, 8), (96, 96, 8, 1))
    assert torch.equal(output_mask(x.untyped_storage().nbytes(), [x, x4]), output_mask(x.untyped_storage().nbytes(), [x]))
    # partial rows of a 2-byte dtype: exactly the bytes of the elements
    part = x[3:5, 1:3]
    mb = output_mask(x.untyped_storage().nbytes(), [part]).view(12, 8, 2)
    assert mb[3:5, 1:3].all() and int(mb.sum()) == 2 * 2 * 2
    # a tuple description, and a snapshot's pre-launch view of a slice
    assert torch.equal(output_mask(nb, [(torch.float32, hi.shape, hi.stride(), hi.storage_offset())]), output_mask(nb, [hi]))
    pre = storage_bytes(buf).clone().view(torch.float32).as_strided(lo.shape, lo.stride(), lo.storage_offset())
    lo.fill_(1.0)
    assert (pre == 0).all() and (lo == 1).all() and not hi.any()


def test_every_launcher_has_a_reference_or_is_listed():
    assert set(leaf_launchers()) == set(CHECKS) | set(NO_REFERENCE), sorted(set(leaf_launchers()) ^ (set(CHECKS) | set(NO_REFERENCE)))

"""CPU oracle for Unicorn's per-frame inference hot path — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A plain fp32 PyTorch/NumPy restatement of the reference's algorithm (MasterBin-IIAU/Unicorn @ 4da9079), written
functionally over a reference-format state_dict.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
`--impl reference` leg may import it; the product (unicorn_b200/) never does.

Parity status: PINNED against the reference's own modules, imported in the build container
(oracle/ref_import.py) — tests/golden/make_golden.py runs both on the same seeded weights/inputs and
tests/test_oracle_golden.py re-checks this file against the committed outputs on any machine.
The MSDA core is additionally pinned to the reference's only known-answer test (unicorn/models/ops/test.py:21-56,
seed 3 shapes) through ms_deform_attn_core_pytorch.  NMS is restated as stable greedy per-class NMS on an exact numpy
emulation of torchvision's CUDA devIoU (fused union, float32 threshold), checked against torchvision.ops.nms on CUDA
(torchvision 0.26) at near-threshold pairs; equal scores are visited in ascending index, which torchvision does not
promise across versions.

Every function cites the reference file:line it follows (paths relative to the reference repo root).
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

# ----------------------------------------------------------------------------------------------- configs
# exps/default/*.py + unicorn/exp/unicorn_track.py:30-52, unicorn_track_mask.py:31-46
CONFIGS = {
    "unicorn_track_tiny": dict(depths=(3, 3, 9, 3), dims=(96, 192, 384, 768), num_classes=8, mask=False),
    "unicorn_track_large": dict(depths=(3, 3, 27, 3), dims=(192, 384, 768, 1536), num_classes=8, mask=False),
    "unicorn_track_large_mot_challenge": dict(depths=(3, 3, 27, 3), dims=(192, 384, 768, 1536), num_classes=1, mask=False),
    "unicorn_track_tiny_mask": dict(depths=(3, 3, 9, 3), dims=(96, 192, 384, 768), num_classes=8, mask=True),
    "unicorn_track_large_mask": dict(depths=(3, 3, 27, 3), dims=(192, 384, 768, 1536), num_classes=8, mask=True),
}
STRIDES = (8, 16, 32)


# ----------------------------------------------------------------------------------------------- backbone
def layernorm_cf(x, w, b, eps=1e-6):
    """channels_first LayerNorm — unicorn/models/backbone/convnext.py:179-184 (biased variance over C)."""
    u = x.mean(1, keepdim=True)
    s = (x - u).pow(2).mean(1, keepdim=True)
    x = (x - u) / torch.sqrt(s + eps)
    return w[:, None, None] * x + b[:, None, None]


def convnext_block(x, sd, p):
    """ConvNeXt Block — convnext.py:41-54: dw7x7 -> LN(eps 1e-6) -> Linear -> GELU(erf) -> Linear -> gamma -> +x."""
    inp = x
    C = x.shape[1]
    x = F.conv2d(x, sd[p + "dwconv.weight"], sd[p + "dwconv.bias"], padding=3, groups=C)
    x = x.permute(0, 2, 3, 1)
    x = F.layer_norm(x, (C,), sd[p + "norm.weight"], sd[p + "norm.bias"], 1e-6)
    x = F.linear(x, sd[p + "pwconv1.weight"], sd[p + "pwconv1.bias"])
    x = F.gelu(x)
    x = F.linear(x, sd[p + "pwconv2.weight"], sd[p + "pwconv2.bias"])
    x = sd[p + "gamma"] * x
    return inp + x.permute(0, 3, 1, 2)


def convnext_features(img, sd, cfg, p="backbone.backbone."):
    """ConvNeXt.forward_features — convnext.py:141-154 (out_indices [1,2,3], out-norms norm1..3 :102-106)."""
    outs = []
    x = img
    for i in range(4):
        d = p + f"downsample_layers.{i}."
        if i == 0:  # stem conv4x4s4 + LN(cf) — convnext.py:77-80
            x = F.conv2d(x, sd[d + "0.weight"], sd[d + "0.bias"], stride=4)
            x = layernorm_cf(x, sd[d + "1.weight"], sd[d + "1.bias"])
        else:  # LN(cf) + conv2x2s2 — convnext.py:82-87
            x = layernorm_cf(x, sd[d + "0.weight"], sd[d + "0.bias"])
            x = F.conv2d(x, sd[d + "1.weight"], sd[d + "1.bias"], stride=2)
        for j in range(cfg["depths"][i]):
            x = convnext_block(x, sd, p + f"stages.{i}.{j}.")
        if i >= 1:
            outs.append(layernorm_cf(x, sd[p + f"norm{i}.weight"], sd[p + f"norm{i}.bias"]))
    return outs  # [s8, s16, s32]


def base_conv(x, sd, p, k, s=1):
    """BaseConv with BN->GN(16, eps 1e-3) — network_blocks.py:29-51; exp/unicorn_track.py:118-122,450-470."""
    x = F.conv2d(x, sd[p + "conv.weight"], None, stride=s, padding=(k - 1) // 2)
    x = F.group_norm(x, 16, sd[p + "bn.weight"], sd[p + "bn.bias"], 1e-3)
    return F.silu(x)


def csp_layer(x, sd, p, n=3):
    """CSPLayer(shortcut=False, n=3) — network_blocks.py:147-185; Bottleneck :79-101 (expansion 1.0, no add)."""
    x1 = base_conv(x, sd, p + "conv1.", 1)
    x2 = base_conv(x, sd, p + "conv2.", 1)
    for i in range(n):
        x1 = base_conv(base_conv(x1, sd, p + f"m.{i}.conv1.", 1), sd, p + f"m.{i}.conv2.", 3)
    return base_conv(torch.cat((x1, x2), 1), sd, p + "conv3.", 1)


def pafpn(feats, sd, p="backbone."):
    """YOLOPAFPNNEW.forward (width 1) — yolo_pafpn_new.py:137-155."""
    x2, x1, x0 = feats
    up = lambda t: F.interpolate(t, scale_factor=2, mode="nearest")  # noqa: E731  (:62)
    fpn_out0 = base_conv(x0, sd, p + "lateral_conv0.", 1)
    f_out0 = csp_layer(torch.cat([up(fpn_out0), x1], 1), sd, p + "C3_p4.")
    fpn_out1 = base_conv(f_out0, sd, p + "reduce_conv1.", 1)
    pan_out2 = csp_layer(torch.cat([up(fpn_out1), x2], 1), sd, p + "C3_p3.")
    p_out1 = base_conv(pan_out2, sd, p + "bu_conv2.", 3, 2)
    pan_out1 = csp_layer(torch.cat([p_out1, fpn_out1], 1), sd, p + "C3_n3.")
    p_out0 = base_conv(pan_out1, sd, p + "bu_conv1.", 3, 2)
    pan_out0 = csp_layer(torch.cat([p_out0, fpn_out0], 1), sd, p + "C3_n4.")
    return (pan_out2, pan_out1, pan_out0)


def pos_embed(sd, h, w):
    """PositionEmbeddingLearned.forward — position_encoding.py:25-36 (+ identity bicubic, unicorn.py:249)."""
    col, row = sd["pos_emb.col_embed.weight"], sd["pos_emb.row_embed.weight"]
    sz = col.shape[0]
    pos = torch.cat([col.unsqueeze(0).repeat(sz, 1, 1), row.unsqueeze(1).repeat(1, sz, 1)], dim=-1)
    pos = pos.permute(2, 0, 1).unsqueeze(0)
    return F.interpolate(pos, (h, w), mode="bilinear", align_corners=False)


def forward_backbone(img, sd, cfg):
    """Unicorn.forward_backbone — unicorn.py:231-258.  Returns (fpn_outs, seq_dict)."""
    feats = convnext_features(img, sd, cfg)
    fpn = pafpn(feats, sd)
    feat = feats[1]
    h, w = feat.shape[-2:]
    return fpn, {"feat": feat, "pos": pos_embed(sd, h, w), "h": h, "w": w}


# ----------------------------------------------------------------------------------------------- interaction
def msda_core(value, shapes, loc, attn):
    """ms_deformable_im2col_gpu_kernel — ops/src/cuda/ms_deform_im2col_cuda.cuh:237-299 with the bilinear gather
    of :33-84: pixel coords h_im = loc_y*H - 0.5, w_im = loc_x*W - 0.5; a sample counts only if -1 < h_im < H and
    -1 < w_im < W; corners outside the map contribute 0.
      value (N,S,M,D), shapes [(H,W)...], loc (N,Lq,M,L,P,2) normalised (x,y), attn (N,Lq,M,L,P) -> (N,Lq,M*D)"""
    N, S, M, D = value.shape
    _, Lq, _, L, P, _ = loc.shape
    out = torch.zeros(N, Lq, M, D, dtype=value.dtype)
    start = 0
    for l, (H, W) in enumerate(shapes):
        v = value[:, start:start + H * W]  # (N,HW,M,D)
        start += H * W
        w_im = loc[:, :, :, l, :, 0] * W - 0.5  # (N,Lq,M,P)
        h_im = loc[:, :, :, l, :, 1] * H - 0.5
        ok = (h_im > -1) & (w_im > -1) & (h_im < H) & (w_im < W)
        h0 = torch.floor(h_im)
        w0 = torch.floor(w_im)
        lh, lw = h_im - h0, w_im - w0
        acc = torch.zeros(N, Lq, M, P, D, dtype=value.dtype)
        for dh, dw, wt in ((0, 0, (1 - lh) * (1 - lw)), (0, 1, (1 - lh) * lw), (1, 0, lh * (1 - lw)), (1, 1, lh * lw)):
            hh, ww = (h0 + dh).long(), (w0 + dw).long()
            inb = ok & (hh >= 0) & (hh < H) & (ww >= 0) & (ww < W)
            idx = (hh.clamp(0, H - 1) * W + ww.clamp(0, W - 1))  # (N,Lq,M,P)
            # gather v[n, idx, m, :]
            idx_e = idx.permute(0, 2, 1, 3).reshape(N, M, Lq * P)  # (N,M,Lq*P)
            vv = v.permute(0, 2, 1, 3)  # (N,M,HW,D)
            g = torch.gather(vv, 2, idx_e.unsqueeze(-1).expand(-1, -1, -1, D)).reshape(N, M, Lq, P, D).permute(0, 2, 1, 3, 4)
            acc = acc + g * (wt * inb)[..., None]
        out = out + (acc * attn[:, :, :, l, :, None]).sum(3)
    return out.reshape(N, Lq, M * D)


def ms_deform_attn(query, ref_points, src, shapes, sd, p, n_heads=8, n_points=4):
    """MSDeformAttn.forward — ops/modules/ms_deform_attn.py:94-115."""
    N, Lq, C = query.shape
    L = len(shapes)
    value = F.linear(src, sd[p + "value_proj.weight"], sd[p + "value_proj.bias"]).view(N, -1, n_heads, C // n_heads)
    off = F.linear(query, sd[p + "sampling_offsets.weight"], sd[p + "sampling_offsets.bias"]).view(N, Lq, n_heads, L, n_points, 2)
    aw = F.linear(query, sd[p + "attention_weights.weight"], sd[p + "attention_weights.bias"]).view(N, Lq, n_heads, L * n_points)
    aw = F.softmax(aw, -1).view(N, Lq, n_heads, L, n_points)
    normalizer = torch.tensor([[w, h] for (h, w) in shapes], dtype=query.dtype)
    loc = ref_points[:, :, None, :, None, :] + off / normalizer[None, None, None, :, None, :]
    out = msda_core(value, shapes, loc, aw)
    return F.linear(out, sd[p + "output_proj.weight"], sd[p + "output_proj.bias"])


def deform_interaction(seq0, seq1, sd):
    """Unicorn.forward_deform_interact — unicorn.py:260-276; DeformableTransformer.forward —
    deformable_transformer.py:58-89; encoder layer :122-131 (post-norm, ReLU FFN); reference points :141-153."""
    srcs, poss = [], []
    for d in (seq0, seq1):
        x = F.conv2d(d["feat"], sd["bottleneck.0.weight"], sd["bottleneck.0.bias"])
        srcs.append(F.group_norm(x, 32, sd["bottleneck.1.weight"], sd["bottleneck.1.bias"], 1e-5))
        poss.append(d["pos"])
    shapes, src_f, pos_f = [], [], []
    for lvl, (s, pe) in enumerate(zip(srcs, poss)):
        bs, c, h, w = s.shape
        shapes.append((h, w))
        src_f.append(s.flatten(2).transpose(1, 2))
        pos_f.append(pe.flatten(2).transpose(1, 2) + sd["transformer.level_embed"][lvl].view(1, 1, -1))
    src = torch.cat(src_f, 1)
    pos = torch.cat(pos_f, 1)
    refs = []
    for (H_, W_) in shapes:  # valid ratios are all 1 (no padding mask)
        ry, rx = torch.meshgrid(torch.linspace(0.5, H_ - 0.5, H_), torch.linspace(0.5, W_ - 0.5, W_), indexing="ij")
        refs.append(torch.stack((rx.reshape(-1) / W_, ry.reshape(-1) / H_), -1)[None])
    ref = torch.cat(refs, 1)[:, :, None].repeat(1, 1, len(shapes), 1)  # (1, S, L, 2)
    p = "transformer.encoder.layers.0."
    src2 = ms_deform_attn(src + pos, ref, src, shapes, sd, p + "self_attn.")
    src = F.layer_norm(src + src2, (256,), sd[p + "norm1.weight"], sd[p + "norm1.bias"], 1e-5)
    ff = F.linear(F.relu(F.linear(src, sd[p + "linear1.weight"], sd[p + "linear1.bias"])), sd[p + "linear2.weight"], sd[p + "linear2.bias"])
    src = F.layer_norm(src + ff, (256,), sd[p + "norm2.weight"], sd[p + "norm2.bias"], 1e-5)
    bs, S, c = src.shape
    half = S // 2
    h, w = seq0["h"], seq0["w"]
    f0 = src[:, :half].permute(0, 2, 1).reshape(bs, c, h, w)
    f1 = src[:, half:].permute(0, 2, 1).reshape(bs, c, h, w)
    return f0, f1


def upsample_embed(feat, sd):
    """Unicorn.forward_upsample — unicorn.py:41-44,311-313."""
    x = F.pixel_shuffle(feat, 2)
    x = F.relu(F.conv2d(x, sd["upsample_layer.1.weight"], sd["upsample_layer.1.bias"], padding=1))
    return F.conv2d(x, sd["upsample_layer.3.weight"], sd["upsample_layer.3.bias"], padding=1)


# ----------------------------------------------------------------------------------------------- correlation
def get_label_map(box_xyxy, H, W):
    """get_label_map — external/lib/test/tracker/unicorn_sot.py:128-139."""
    labels = torch.zeros((1, 1, H, W), dtype=torch.float32)
    x1, y1, x2, y2 = torch.round(torch.as_tensor(box_xyxy, dtype=torch.float32)).int().tolist()
    x1, x2 = max(0, min(x1, W)), max(0, min(x2, W))
    y1, y2 = max(0, min(y1, H)), max(0, min(y2, H))
    labels[0, 0, y1:y2, x1:x2] = 1.0
    return labels


def label_map_s8(box_xyxy, H, W):
    """unicorn_sot.py:52-53: bilinear x1/8, align_corners False -> (K, H/8*W/8)."""
    return F.interpolate(get_label_map(box_xyxy, H, W), scale_factor=1 / 8, mode="bilinear", align_corners=False)[0].flatten(-2)


def corr_propagate(embed_pre, embed_cur, values, half=False):
    """unicorn_sot.py:88-100 / unicorn_vos.py:166-181: S = K^T Q; T = softmax(S, dim=0); pred = V T.
    embed_* (C, N), values (K, N) -> (K, N).  half=True mimics the reference's fp16 casts (rounding only)."""
    keys, cur, vals = embed_pre, embed_cur, values
    if half:
        keys, cur, vals = keys.half().float(), cur.half().float(), vals.half().float()
    simi = keys.transpose(1, 0) @ cur
    if half:
        simi = simi.half().float()
    trans = torch.softmax(simi, dim=0)
    if half:
        trans = trans.half().float()
    out = vals @ trans
    return out.half().float() if half else out


def prior_pyramid(coarse_m):
    """unicorn_sot.py:103-105: (1,K,h,w) -> [x1, x1/2, x1/4] bilinear align_corners False."""
    return (coarse_m,
            F.interpolate(coarse_m, scale_factor=1 / 2, mode="bilinear", align_corners=False),
            F.interpolate(coarse_m, scale_factor=1 / 4, mode="bilinear", align_corners=False))


# ----------------------------------------------------------------------------------------------- head
def head_forward(fpn, priors, sd, cfg, mode, decode=True, return_feats=False):
    """UnicornHead.forward eval branch — unicorn_head.py:267-336,430-439 and decode_outputs :467-482.
    Returns (1, sum(hw), 5+ncls) rows [cx,cy,w,h,obj,cls...]."""
    outs, hw, reg_feats = [], [], []
    for k in range(3):
        p = "head."
        x = base_conv(fpn[k], sd, p + f"stems.{k}.", 1)
        x = x + priors[k] * sd[p + f"beta_{k}"]  # :272-275 (beta indexed by level k)
        for n in range(3):
            x = convnext_block(x, sd, p + f"att_layers.{k}.{n}.")
        cls_feat, reg_feat = x, x
        for i in range(4):
            cls_feat = base_conv(cls_feat, sd, p + f"cls_convs.{k}.{i}.", 3)
            reg_feat = base_conv(reg_feat, sd, p + f"reg_convs.{k}.{i}.", 3)
        sfx = "_sot" if mode == "sot" else ""
        cls_o = F.conv2d(cls_feat, sd[p + f"cls_preds{sfx}.{k}.weight"], sd[p + f"cls_preds{sfx}.{k}.bias"])
        reg_o = F.conv2d(reg_feat, sd[p + f"reg_preds{sfx}.{k}.weight"], sd[p + f"reg_preds{sfx}.{k}.bias"])
        obj_o = F.conv2d(reg_feat, sd[p + f"obj_preds{sfx}.{k}.weight"], sd[p + f"obj_preds{sfx}.{k}.bias"])
        outs.append(torch.cat([reg_o, obj_o.sigmoid(), cls_o.sigmoid()], 1))
        hw.append(outs[-1].shape[-2:])
        reg_feats.append(reg_feat)
    out = torch.cat([x.flatten(start_dim=2) for x in outs], dim=2).permute(0, 2, 1).contiguous()
    if decode:
        grids, strides = [], []
        for (hs, ws), s in zip(hw, STRIDES):
            yv, xv = torch.meshgrid(torch.arange(hs), torch.arange(ws), indexing="ij")
            grids.append(torch.stack((xv, yv), 2).view(1, -1, 2).float())
            strides.append(torch.full((1, hs * ws, 1), float(s)))
        grids, strides = torch.cat(grids, 1), torch.cat(strides, 1)
        out[..., :2] = (out[..., :2] + grids) * strides
        out[..., 2:4] = torch.exp(out[..., 2:4]) * strides
    if return_feats:
        return out, reg_feats
    return out


def whole_forward(img, sd, cfg):
    """Unicorn.forward(mode="whole") — unicorn.py:133-139: backbone + head on all-zero priors with the MOT prediction set.
    Returns (head output, seq_dict); for a mask model the head output is UnicornHeadMask's tuple (head_forward_mask)."""
    fpn, seq = forward_backbone(img, sd, cfg)
    bs, _, H, W = img.shape
    zeros = tuple(torch.zeros(bs, 1, H // s, W // s) for s in STRIDES)
    if cfg["mask"]:
        return head_forward_mask(fpn, zeros, sd, cfg, "mot"), seq
    return head_forward(fpn, zeros, sd, cfg, "mot"), seq


# ----------------------------------------------------------------------------------------------- post
def box_iou_np(a, b):
    area_a = (a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1])
    area_b = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
    lt = np.maximum(a[:, None, :2], b[None, :, :2])
    rb = np.minimum(a[:, None, 2:], b[None, :, 2:])
    wh = np.clip(rb - lt, 0, None)
    inter = wh[..., 0] * wh[..., 1]
    return inter / (area_a[:, None] + area_b[None, :] - inter)


def fma32(a, b, c):
    """fmaf(a, b, c) of float32 arrays: a * b + c rounded once to float32.  The float64 product of two floats is exact; the
    float64 sum s is off by e (TwoSum: s + e == a * b + c exactly), which changes the float32 rounding only when s is a float32
    midpoint, where the exact sum lies on the side of e."""
    a, b, c = (np.asarray(v, dtype=np.float32).astype(np.float64) for v in (a, b, c))
    p = a * b
    s = p + c
    t = s - p
    e = (p - (s - t)) + (c - t)
    r = s.astype(np.float32)
    r64 = r.astype(np.float64)
    up = s > r64
    other = np.nextafter(r, np.where(up, np.float32(np.inf), np.float32(-np.inf)))
    mid = (s != r64) & ((r64 + other.astype(np.float64)) * 0.5 == s)
    return np.where(mid & (e != 0) & ((e > 0) == up), other, r)


def dev_iou(a, b):
    """IoU of boxes a (earlier in the score order) and b (later), xyxy float32 [..., 4], broadcast: torchvision's CUDA devIoU
    (csrc/ops/cuda/nms_kernel.cu) as nvcc compiles it: rounded widths, heights, intersection and a's area, b's area fused into
    the union, union = fmaf(wb, hb, area_a) - inter, an IEEE divide."""
    f = np.float32
    a, b = np.asarray(a, dtype=f), np.asarray(b, dtype=f)
    w = np.maximum(np.minimum(a[..., 2], b[..., 2]) - np.maximum(a[..., 0], b[..., 0]), f(0))
    h = np.maximum(np.minimum(a[..., 3], b[..., 3]) - np.maximum(a[..., 1], b[..., 1]), f(0))
    inter = w * h
    sa = (a[..., 2] - a[..., 0]) * (a[..., 3] - a[..., 1])
    union = fma32(b[..., 2] - b[..., 0], b[..., 3] - b[..., 1], sa) - inter
    with np.errstate(divide="ignore", invalid="ignore"):
        return inter / union


def box_iou_f32(a, b, plus_one=False):
    """[N, M] IoU with every float32 step rounded on its own: torchvision.ops.box_iou's separate torch ops (plus_one=False),
    and the same order with + 1 after each difference, the inclusive-pixel convention of cython_bbox.bbox_overlaps."""
    f = np.float32
    a, b = np.asarray(a, dtype=f), np.asarray(b, dtype=f)
    one = f(1) if plus_one else f(0)
    area_a = ((a[:, 2] - a[:, 0]) + one) * ((a[:, 3] - a[:, 1]) + one)
    area_b = ((b[:, 2] - b[:, 0]) + one) * ((b[:, 3] - b[:, 1]) + one)
    lt = np.maximum(a[:, None, :2], b[None, :, :2])
    rb = np.minimum(a[:, None, 2:], b[None, :, 2:])
    wh = np.maximum((rb - lt) + one, f(0))
    inter = wh[..., 0] * wh[..., 1]
    with np.errstate(divide="ignore", invalid="ignore"):
        return inter / ((area_a[:, None] + area_b[None, :]) - inter)


def nms_greedy(boxes, scores, thr):
    """torchvision.ops.nms on CUDA: visit in descending score (equal scores in ascending index), a kept box suppresses every
    later box with dev_iou(kept, later) > float32(thr)."""
    boxes = np.asarray(boxes, dtype=np.float32)
    order = np.argsort(-np.asarray(scores, dtype=np.float32), kind="stable")
    thr = np.float32(thr)
    keep = []
    suppressed = np.zeros(len(order), dtype=bool)
    for ii, i in enumerate(order):
        if suppressed[ii]:
            continue
        keep.append(i)
        suppressed[ii + 1:] |= dev_iou(boxes[i], boxes[order[ii + 1:]]) > thr
    return np.asarray(keep, dtype=np.int64)


def postprocess(prediction, num_classes, conf_thre=0.7, nms_thre=0.45):
    """unicorn/utils/boxes.py:33-77 (class-aware batched_nms; output sorted by descending score).
    prediction (1, A, 5+ncls) decoded cxcywh.  Returns list[Tensor(M,7) | None] with rows
    (x1,y1,x2,y2,obj,cls_conf,cls_id)."""
    pred = prediction.clone()
    box = pred.new_zeros(pred.shape)
    box[:, :, 0] = pred[:, :, 0] - pred[:, :, 2] / 2
    box[:, :, 1] = pred[:, :, 1] - pred[:, :, 3] / 2
    box[:, :, 2] = pred[:, :, 0] + pred[:, :, 2] / 2
    box[:, :, 3] = pred[:, :, 1] + pred[:, :, 3] / 2
    pred[:, :, :4] = box[:, :, :4]
    output = [None for _ in range(len(pred))]
    for i, ip in enumerate(pred):
        class_conf, class_pred = torch.max(ip[:, 5:5 + num_classes], 1, keepdim=True)
        mask = (ip[:, 4] * class_conf.squeeze(1) >= conf_thre)
        det = torch.cat((ip[:, :5], class_conf, class_pred.float()), 1)[mask]
        if not det.size(0):
            continue
        scores = (det[:, 4] * det[:, 5]).numpy()
        boxes = det[:, :4].numpy()
        cls = det[:, 6].numpy()
        keep_all = []
        for c in np.unique(cls):
            idx = np.nonzero(cls == c)[0]
            k = nms_greedy(boxes[idx], scores[idx], nms_thre)
            keep_all.append(idx[k])
        keep = np.concatenate(keep_all)
        keep = keep[np.argsort(-scores[keep], kind="stable")]  # batched_nms returns score-sorted indices
        output[i] = det[torch.from_numpy(keep)]
    return output


# ----------------------------------------------------------------------------------------------- SOT driver
class SOTOracle:
    """UnicornSOTTrack.initialize/track — external/lib/test/tracker/unicorn_sot.py:39-109 on pre-processed
    frames (1,3,H,W) fp32 BGR 0..255 (PreprocessorX output)."""

    def __init__(self, sd, cfg_name, conf=0.001, nms=0.65, half_corr=False):
        self.sd, self.cfg = sd, CONFIGS[cfg_name]
        self.conf, self.nms, self.half_corr = conf, nms, half_corr

    @torch.no_grad()
    def initialize(self, ref_frame, init_box_xyxy):
        _, self.pre = forward_backbone(ref_frame, self.sd, self.cfg)
        H, W = ref_frame.shape[-2:]
        self.dh, self.dw = self.pre["h"] * 2, self.pre["w"] * 2
        self.lbs_pre = label_map_s8(init_box_xyxy, H, W)

    @torch.no_grad()
    def track(self, cur_frame, stages=None):
        fpn, cur = forward_backbone(cur_frame, self.sd, self.cfg)
        f_pre, f_cur = deform_interaction(self.pre, cur, self.sd)
        e_pre, e_cur = upsample_embed(f_pre, self.sd), upsample_embed(f_cur, self.sd)
        pred = corr_propagate(e_pre.flatten(-2)[0], e_cur.flatten(-2)[0], self.lbs_pre, half=self.half_corr)
        coarse = pred.view(1, -1, self.dh, self.dw)
        pri = prior_pyramid(coarse)
        out = head_forward(fpn, pri, self.sd, self.cfg, "sot")
        dets = postprocess(out, 1, self.conf, self.nms)[0]
        if stages is not None:
            stages.update(fpn=fpn, feat=cur["feat"], pos=cur["pos"], inter_pre=f_pre, inter_cur=f_cur, embed_pre=e_pre,
                          embed_cur=e_cur, coarse=coarse, head=out, dets=dets)
        return dets


# ----------------------------------------------------------------------------------------------- mask head (config 4)
def aligned_bilinear(t, factor):
    """condinst/comm.py:5-27 (== utils/boxes.py:212-234)."""
    if factor == 1:
        return t
    h, w = t.shape[2:]
    t = F.pad(t, pad=(0, 1, 0, 1), mode="replicate")
    oh, ow = factor * h + 1, factor * w + 1
    t = F.interpolate(t, size=(oh, ow), mode="bilinear", align_corners=True)
    t = F.pad(t, pad=(factor // 2, 0, factor // 2, 0), mode="replicate")
    return t[:, :, :oh - 1, :ow - 1]


def _conv_gn_relu(x, sd, p):
    """conv_with_kaiming_uniform("BN", activation=True) after BN->GN16 (eps 1e-3): conv3x3 (no bias) -> GN -> ReLU
    (condinst/conv_with_kaiming_uniform.py:8-50, exp/unicorn_track.py:118-122,450-470)."""
    x = F.conv2d(x, sd[p + "0.weight"], None, padding=1)
    return F.relu(F.group_norm(x, 16, sd[p + "1.weight"], sd[p + "1.bias"], 1e-3))


def mask_branch(fpn, sd, p="head.mask_branch."):
    """MaskBranch.forward, use_raft=True (condinst/mask_branch.py:77-96,158-162) -> (mask_feats (1,8,h,w), up_masks (1,144,h,w))."""
    x = _conv_gn_relu(fpn[0], sd, p + "refine.0.")
    for i in (1, 2):
        xp = _conv_gn_relu(fpn[i], sd, p + f"refine.{i}.")
        x = x + aligned_bilinear(xp, x.shape[2] // xp.shape[2])
    t = x
    for i in range(4):
        t = _conv_gn_relu(t, sd, p + f"tower.{i}.")
    mask_feats = F.conv2d(t, sd[p + "tower.4.weight"], sd[p + "tower.4.bias"])
    u = F.relu(F.conv2d(x, sd[p + "up_mask_layer.0.weight"], sd[p + "up_mask_layer.0.bias"], padding=1))
    up_masks = F.conv2d(u, sd[p + "up_mask_layer.2.weight"], sd[p + "up_mask_layer.2.bias"])
    return mask_feats, up_masks


def head_forward_mask(fpn, priors, sd, cfg, mode):
    """UnicornHeadMask.forward eval (unicorn_head_mask.py:280-343,451-471) + decode_outputs (:502-519).
    Returns outputs (1,A,5+ncls), locations (A,2), dynamic_params (1,A,169), fpn_levels (1,A), mask_feats, up_masks."""
    out, reg_feats = head_forward(fpn, priors, sd, cfg, mode, decode=True, return_feats=True)
    dyn, lvls, locs = [], [], []
    for k in range(3):
        d = F.conv2d(reg_feats[k], sd[f"head.controllers.{k}.weight"], sd[f"head.controllers.{k}.bias"], padding=1)
        dyn.append(d.flatten(-2).permute(0, 2, 1))
        lvls.append(torch.full((1, d.shape[2] * d.shape[3]), k))
        hs, ws = d.shape[-2:]
        yv, xv = torch.meshgrid(torch.arange(hs), torch.arange(ws), indexing="ij")
        locs.append((torch.stack((xv, yv), 2).view(-1, 2).float() + 0.5) * STRIDES[k])
    mf, um = mask_branch(fpn, sd)
    return out, torch.cat(locs, 0), torch.cat(dyn, 1), torch.cat(lvls, 1), mf, um


def dynamic_masks(mask_feats, params, inst_locs, inst_levels, up_masks, up_rate=4, soi=(64.0, 128.0, 256.0, 512.0, 1024.0)):
    """DynamicMaskHead.__call__ eval (condinst/dynamic_mask_head.py:172-225,159-170,284): -> (N,1,up*h,up*w) sigmoid."""
    _, C, H, W = mask_feats.shape
    n = params.shape[0]
    sx = torch.arange(0, W * 8, step=8, dtype=torch.float32)
    sy = torch.arange(0, H * 8, step=8, dtype=torch.float32)
    yy, xx = torch.meshgrid(sy, sx, indexing="ij")
    locations = torch.stack((xx.reshape(-1), yy.reshape(-1)), dim=1) + 4  # compute_locations (comm.py:30-45)
    rel = (inst_locs.reshape(-1, 1, 2) - locations.reshape(1, -1, 2)).permute(0, 2, 1).float()
    rel = rel / torch.tensor(soi)[inst_levels.long()].reshape(-1, 1, 1)
    x = torch.cat([rel, mask_feats[0].reshape(1, C, H * W).expand(n, -1, -1)], dim=1)  # (N,10,HW)
    w0, w1, w2, b0, b1, b2 = torch.split_with_sizes(params, [80, 64, 8, 8, 8, 1], dim=1)  # parse_dynamic_params :61-87
    x = F.relu(torch.bmm(w0.reshape(n, 8, 10), x) + b0.reshape(n, 8, 1))
    x = F.relu(torch.bmm(w1.reshape(n, 8, 8), x) + b1.reshape(n, 8, 1))
    logits = (torch.bmm(w2.reshape(n, 1, 8), x) + b2.reshape(n, 1, 1)).reshape(n, 1, H, W)
    m = torch.softmax(up_masks.view(1, 1, 9, up_rate, up_rate, H, W), dim=2)  # upsample_preds :159-170
    up = F.unfold(logits, [3, 3], padding=1).view(n, 1, 9, 1, 1, H, W)
    up = torch.sum(m * up, dim=2).permute(0, 1, 4, 2, 5, 3).reshape(n, 1, up_rate * H, up_rate * W)
    return up.sigmoid()


def postprocess_inst(pred, locations, dyn, levels, mask_feats, up_masks, num_classes, conf_thre, nms_thre, d_rate=2, max_masks=None):
    """utils/boxes.py:80-152 for one image: (dets (M,7), masks (min(M,max_masks),1,H,W)); max_masks limits how many
    of the (score-ordered) instances get a mask (the VOS driver only reads the first, unicorn_vos.py:121-149)."""
    p = pred.clone()
    box = p.new_zeros(p.shape)
    box[:, :, 0] = p[:, :, 0] - p[:, :, 2] / 2
    box[:, :, 1] = p[:, :, 1] - p[:, :, 3] / 2
    box[:, :, 2] = p[:, :, 0] + p[:, :, 2] / 2
    box[:, :, 3] = p[:, :, 1] + p[:, :, 3] / 2
    p[:, :, :4] = box[:, :, :4]
    ip = p[0]
    cc, cp = torch.max(ip[:, 5:5 + num_classes], 1, keepdim=True)
    mask = ip[:, 4] * cc.squeeze(1) >= conf_thre
    det = torch.cat((ip[:, :5], cc, cp.float()), 1)[mask]
    if det.shape[0] == 0:
        return None, None
    scores = (det[:, 4] * det[:, 5]).numpy()
    keep_all = []
    for c in np.unique(det[:, 6].numpy()):
        idx = np.nonzero(det[:, 6].numpy() == c)[0]
        keep_all.append(idx[nms_greedy(det[idx, :4].numpy(), scores[idx], nms_thre)])
    keep = np.concatenate(keep_all)
    keep = torch.from_numpy(keep[np.argsort(-scores[keep], kind="stable")])
    det = det[keep]
    k = keep if max_masks is None else keep[:max_masks]
    masks = dynamic_masks(mask_feats, dyn[0][mask][k], locations[mask][k], levels[0][mask][k], up_masks, up_rate=8 // d_rate)
    return det, aligned_bilinear(masks, d_rate)


# ----------------------------------------------------------------------------------------------- VOS driver (config 4)
class VOSOracle:
    """UnicornVOSTrack — external/lib/test/tracker/unicorn_vos.py: initialize :43-69, track :71-127 (groups of later objects
    :79-98, soft aggregation :100-121), get_mask_results :129-155, get_det_results :157-201 — on pre-processed frames
    (1,3,H,W) fp32 BGR 0..255, fp32 correlation (half_corr mimics the reference's fp16 casts)."""

    def __init__(self, sd, cfg_name, conf=0.001, nms=0.65, d_rate=2, half_corr=False):
        self.sd, self.cfg = sd, CONFIGS[cfg_name]
        self.conf, self.nms, self.d_rate, self.half_corr = conf, nms, d_rate, half_corr

    @torch.no_grad()
    def initialize(self, ref_frame, boxes_xyxy, orig_size=None, r=1.0):
        _, pre = forward_backbone(ref_frame, self.sd, self.cfg)
        self.in_size = tuple(ref_frame.shape[-2:])
        self.H, self.W = orig_size if orig_size is not None else self.in_size
        self.r = r
        self.dh, self.dw = pre["h"] * 2, pre["w"] * 2
        self.groups = [(pre, list(boxes_xyxy.keys()))]
        self.lbs = {o: label_map_s8(b, *self.in_size) for o, b in boxes_xyxy.items()}

    def _group_results(self, fpn, cur, pre, ids):  # get_det_results + get_mask_results
        f_pre, f_cur = deform_interaction(pre, cur, self.sd)
        e_pre, e_cur = upsample_embed(f_pre, self.sd), upsample_embed(f_cur, self.sd)
        out = {}
        for o in ids:
            pred = corr_propagate(e_pre.flatten(-2)[0], e_cur.flatten(-2)[0], self.lbs[o], half=self.half_corr)
            coarse = pred.view(1, -1, self.dh, self.dw).float()
            outs, locs, dyn, lvls, mf, um = head_forward_mask(fpn, prior_pyramid(coarse), self.sd, self.cfg, "sot")
            det, masks = postprocess_inst(outs, locs, dyn, lvls, mf, um, 1, self.conf, self.nms, d_rate=self.d_rate, max_masks=1)
            soft = np.zeros((self.H, self.W), dtype=np.float32)
            if det is not None:
                m = F.interpolate(masks, scale_factor=1 / self.r, mode="bilinear", align_corners=False)[:, 0, :self.H, :self.W]
                soft[:m.shape[1], :m.shape[2]] = m[0].numpy()
            out[o] = dict(det=None if det is None else det[0], soft=soft, coarse=coarse, head=outs, mask=None if det is None else masks[0, 0])
        return out

    @torch.no_grad()
    def track(self, cur_frame, new_boxes_xyxy=None, init_mask=None):
        """-> (segmentation uint8 (H,W), {obj_id: dict(det, soft, ...)}); new objects: boxes in resized-image coordinates and the
        label map `init_mask` (H,W) of this frame."""
        fpn, cur = forward_backbone(cur_frame, self.sd, self.cfg)
        res = {}
        for pre, ids in self.groups:
            res.update(self._group_results(fpn, cur, pre, ids))
        cur_ids = [o for _, ids in self.groups for o in ids]
        if new_boxes_xyxy:
            self.groups.append((cur, list(new_boxes_xyxy.keys())))
            for o, b in new_boxes_xyxy.items():
                self.lbs[o] = label_map_s8(b, *self.in_size)
                res[o] = dict(det=None, soft=(np.asarray(init_mask) == int(o)))
                cur_ids.append(o)
        merge = np.zeros((self.H, self.W, max(int(o) for o in cur_ids) + 1))  # :106-117
        tmp = []
        for o in cur_ids:
            merge[:, :, int(o)] = res[o]["soft"]
            tmp.append(res[o]["soft"])
        merge[:, :, 0] = np.prod(1 - np.stack(tmp, axis=-1), axis=-1, keepdims=False)
        final = np.argmax(merge, axis=-1)
        seg = np.zeros((self.H, self.W), dtype=np.uint8)
        for o in cur_ids:
            seg[final == int(o)] = int(o)
        return seg, res

"""Weight interface of the Unicorn tracking models: the reference's state_dict key set and a deterministic
random initialiser for it (there are no checkpoints offline — benchmarks and tests use seeded weights).

Key names/shapes follow the reference modules (unicorn/models/unicorn.py:28-44, backbone/convnext.py:71-106,
backbone/yolo_pafpn_new.py:62-111, unicorn_head.py:58-228, deformable_transformer.py:22-37,99-114,
ops/modules/ms_deform_attn.py:55-58, condinst/mask_branch.py:17-70, unicorn_head_mask.py controllers) and are
pinned to manifests dumped from the reference itself (tests/golden/manifest_*.json, tests/test_weights.py).
"""
import math
import zlib
from collections import OrderedDict

import torch

CONFIGS = {
    "unicorn_track_tiny": dict(depths=(3, 3, 9, 3), dims=(96, 192, 384, 768), num_classes=8, mask=False),
    "unicorn_track_large": dict(depths=(3, 3, 27, 3), dims=(192, 384, 768, 1536), num_classes=8, mask=False),
    "unicorn_track_large_mot_challenge": dict(depths=(3, 3, 27, 3), dims=(192, 384, 768, 1536), num_classes=1, mask=False),
    "unicorn_track_tiny_mask": dict(depths=(3, 3, 9, 3), dims=(96, 192, 384, 768), num_classes=8, mask=True),
    "unicorn_track_large_mask": dict(depths=(3, 3, 27, 3), dims=(192, 384, 768, 1536), num_classes=8, mask=True),
    # the released MOTS20 model: the 1-class head of *_mot_challenge with the mask head of *_mask
    "unicorn_track_large_mot_challenge_mask": dict(depths=(3, 3, 27, 3), dims=(192, 384, 768, 1536), num_classes=1, mask=True),
    # exps/default/unicorn_track_r50*.py: torchvision ResNet-50 (v1.5 Bottlenecks); dims = the stage output widths (4 x 64/128/256/512)
    "unicorn_track_r50": dict(backbone="resnet50", depths=(3, 4, 6, 3), dims=(256, 512, 1024, 2048), num_classes=8, mask=False),
    "unicorn_track_r50_mask": dict(backbone="resnet50", depths=(3, 4, 6, 3), dims=(256, 512, 1024, 2048), num_classes=8, mask=True),
    # the COCO detectors (exps/default/unicorn_det_*_800x1280.py, YOLOX + YOLOXHeadDet): backbone, neck and an 80-class head without the
    # prior term, the SOT predictors and the interaction modules; the first stage of the tracking models of the same backbone
    "unicorn_det_convnext_tiny": dict(task="det", depths=(3, 3, 9, 3), dims=(96, 192, 384, 768), num_classes=80, mask=False),
    "unicorn_det_convnext_large": dict(task="det", depths=(3, 3, 27, 3), dims=(192, 384, 768, 1536), num_classes=80, mask=False),
    "unicorn_det_r50": dict(task="det", backbone="resnet50", depths=(3, 4, 6, 3), dims=(256, 512, 1024, 2048), num_classes=80, mask=False),
    # the COCO instance segmenter (exps/default/unicorn_inst_convnext_tiny_800x1280.py, YOLOX + YOLOXHeadDetMask, CondInst): the
    # ConvNeXt-T detector plus the per-level controllers and the RAFT mask branch of the tracking *_mask heads
    "unicorn_inst_convnext_tiny": dict(task="det", depths=(3, 3, 9, 3), dims=(96, 192, 384, 768), num_classes=80, mask=True),
}
for _c in CONFIGS.values():
    _c.setdefault("task", "track")
    _c.setdefault("backbone", "convnext")
    _c["in_channels"] = tuple(_c["dims"][1:])  # channels of the s8 / s16 / s32 maps the neck, heads and interaction read


def param_shapes(cfg_name):
    """OrderedDict name -> shape, in the reference's state_dict order."""
    cfg = CONFIGS[cfg_name]
    depths, dims, ncls = cfg["depths"], cfg["dims"], cfg["num_classes"]
    inc = cfg["in_channels"]
    S = OrderedDict()

    def bn(p, c):  # BatchNorm2d, kept as BN in the ResNet backbone (exp/unicorn_track.py:147-153)
        S[p + "weight"] = (c,); S[p + "bias"] = (c,)
        S[p + "running_mean"] = (c,); S[p + "running_var"] = (c,); S[p + "num_batches_tracked"] = ()

    b = "backbone.backbone."
    if cfg["backbone"] == "resnet50":  # backbone/resnet.py:127-204 (no fc: out_indices [1, 2, 3])
        S[b + "conv1.weight"] = (64, 3, 7, 7)
        bn(b + "bn1.", 64)
        cin = 64
        for i, n in enumerate(depths):
            w = 64 << i
            for j in range(n):
                p = b + f"layer{i + 1}.{j}."
                S[p + "conv1.weight"] = (w, cin, 1, 1); bn(p + "bn1.", w)
                S[p + "conv2.weight"] = (w, w, 3, 3); bn(p + "bn2.", w)
                S[p + "conv3.weight"] = (4 * w, w, 1, 1); bn(p + "bn3.", 4 * w)
                if j == 0:
                    S[p + "downsample.0.weight"] = (4 * w, cin, 1, 1); bn(p + "downsample.1.", 4 * w)
                cin = 4 * w
    else:
        _convnext_shapes(S, b, depths, dims)
    _neck_and_heads(S, inc, ncls, cfg["mask"], cfg["task"] == "det")
    return S


def _convnext_block(S, p, d):
    S[p + "gamma"] = (d,)
    S[p + "dwconv.weight"] = (d, 1, 7, 7); S[p + "dwconv.bias"] = (d,)
    S[p + "norm.weight"] = (d,); S[p + "norm.bias"] = (d,)
    S[p + "pwconv1.weight"] = (4 * d, d); S[p + "pwconv1.bias"] = (4 * d,)
    S[p + "pwconv2.weight"] = (d, 4 * d); S[p + "pwconv2.bias"] = (d,)


def _convnext_shapes(S, b, depths, dims):
    S[b + "downsample_layers.0.0.weight"] = (dims[0], 3, 4, 4); S[b + "downsample_layers.0.0.bias"] = (dims[0],)
    S[b + "downsample_layers.0.1.weight"] = (dims[0],); S[b + "downsample_layers.0.1.bias"] = (dims[0],)
    for i in range(1, 4):
        S[b + f"downsample_layers.{i}.0.weight"] = (dims[i - 1],); S[b + f"downsample_layers.{i}.0.bias"] = (dims[i - 1],)
        S[b + f"downsample_layers.{i}.1.weight"] = (dims[i], dims[i - 1], 2, 2); S[b + f"downsample_layers.{i}.1.bias"] = (dims[i],)
    for i in range(4):
        for j in range(depths[i]):
            _convnext_block(S, b + f"stages.{i}.{j}.", dims[i])
    for i in range(1, 4):
        S[b + f"norm{i}.weight"] = (dims[i],); S[b + f"norm{i}.bias"] = (dims[i],)


def _neck_and_heads(S, inc, ncls, mask, det=False):
    """The neck and the head; det=True: YOLOXHeadDet (yolo_head_det.py:53-190), the head without the prior scales (`beta_*`), the
    SOT predictors and the interaction / upsampling modules that follow it."""
    def baseconv(p, cin, cout, k):
        S[p + "conv.weight"] = (cout, cin, k, k)
        S[p + "bn.weight"] = (cout,); S[p + "bn.bias"] = (cout,)

    def csp(p, cin, cout, n=3):
        h = cout // 2
        baseconv(p + "conv1.", cin, h, 1)
        baseconv(p + "conv2.", cin, h, 1)
        baseconv(p + "conv3.", 2 * h, cout, 1)
        for i in range(n):
            baseconv(p + f"m.{i}.conv1.", h, h, 1)
            baseconv(p + f"m.{i}.conv2.", h, h, 3)

    p = "backbone."
    baseconv(p + "lateral_conv0.", inc[2], inc[1], 1)
    csp(p + "C3_p4.", 2 * inc[1], inc[1])
    baseconv(p + "reduce_conv1.", inc[1], inc[0], 1)
    csp(p + "C3_p3.", 2 * inc[0], inc[0])
    baseconv(p + "bu_conv2.", inc[0], inc[0], 3)
    csp(p + "C3_n3.", 2 * inc[0], inc[1])
    baseconv(p + "bu_conv1.", inc[1], inc[1], 3)
    csp(p + "C3_n4.", 2 * inc[1], inc[2])
    h = "head."
    for k in range(3 if not det else 0):
        S[h + f"beta_{k}"] = (256, 1, 1)
    for k in range(3):
        for i in range(4):
            baseconv(h + f"cls_convs.{k}.{i}.", 256, 256, 3)
    for k in range(3):
        for i in range(4):
            baseconv(h + f"reg_convs.{k}.{i}.", 256, 256, 3)
    preds = (("cls_preds", ncls), ("reg_preds", 4), ("obj_preds", 1))
    for name, co in preds + (() if det else (("cls_preds_sot", 1), ("obj_preds_sot", 1), ("reg_preds_sot", 4))):
        for k in range(3):
            S[h + f"{name}.{k}.weight"] = (co, 256, 1, 1); S[h + f"{name}.{k}.bias"] = (co,)
    if mask:
        S[h + "mask_head.sizes_of_interest"] = (5,)
        S[h + "mask_head._iter"] = (1,)
        for k in range(3):
            S[h + f"mask_branch.refine.{k}.0.weight"] = (128, inc[k], 3, 3)
            S[h + f"mask_branch.refine.{k}.1.weight"] = (128,); S[h + f"mask_branch.refine.{k}.1.bias"] = (128,)
        for i in range(4):
            S[h + f"mask_branch.tower.{i}.0.weight"] = (128, 128, 3, 3)
            S[h + f"mask_branch.tower.{i}.1.weight"] = (128,); S[h + f"mask_branch.tower.{i}.1.bias"] = (128,)
        S[h + "mask_branch.tower.4.weight"] = (8, 128, 1, 1); S[h + "mask_branch.tower.4.bias"] = (8,)
        S[h + "mask_branch.up_mask_layer.0.weight"] = (128, 128, 3, 3); S[h + "mask_branch.up_mask_layer.0.bias"] = (128,)
        S[h + "mask_branch.up_mask_layer.2.weight"] = (144, 128, 1, 1); S[h + "mask_branch.up_mask_layer.2.bias"] = (144,)
        for k in range(3):
            S[h + f"controllers.{k}.weight"] = (169, 256, 3, 3); S[h + f"controllers.{k}.bias"] = (169,)
    for k in range(3):
        baseconv(h + f"stems.{k}.", inc[k], 256, 1)
    for k in range(3):
        for n in range(3):
            _convnext_block(S, h + f"att_layers.{k}.{n}.", 256)
    if det:
        return
    S["bottleneck.0.weight"] = (256, inc[1], 1, 1); S["bottleneck.0.bias"] = (256,)
    S["bottleneck.1.weight"] = (256,); S["bottleneck.1.bias"] = (256,)
    S["upsample_layer.1.weight"] = (256, 64, 3, 3); S["upsample_layer.1.bias"] = (256,)
    S["upsample_layer.3.weight"] = (128, 256, 3, 3); S["upsample_layer.3.bias"] = (128,)
    S["pos_emb.row_embed.weight"] = (40, 128); S["pos_emb.col_embed.weight"] = (40, 128)
    S["transformer.level_embed"] = (2, 256)
    t = "transformer.encoder.layers.0."
    for name, co in (("sampling_offsets", 128), ("attention_weights", 64), ("value_proj", 256), ("output_proj", 256)):
        S[t + f"self_attn.{name}.weight"] = (co, 256); S[t + f"self_attn.{name}.bias"] = (co,)
    S[t + "norm1.weight"] = (256,); S[t + "norm1.bias"] = (256,)
    S[t + "linear1.weight"] = (1024, 256); S[t + "linear1.bias"] = (1024,)
    S[t + "linear2.weight"] = (256, 1024); S[t + "linear2.bias"] = (256,)
    S[t + "norm2.weight"] = (256,); S[t + "norm2.bias"] = (256,)


def _gen(name, seed):
    return torch.Generator(device="cpu").manual_seed((zlib.crc32(name.encode()) ^ (seed * 0x9E3779B1)) & 0x7FFFFFFF)


def make_state_dict(cfg_name, seed=0):
    """Deterministic, well-conditioned random weights keyed like the reference state_dict (fp32, CPU).

    Unlike the reference's init (zero attention/offset weights, -4.6 prediction biases, unit layer scales) every
    parameter is perturbed so that every kernel's output depends on its inputs and detections exist — the caveats
    listed in SURVEY.md §8(c) — while activations stay O(1) through 36 residual blocks.  BatchNorm buffers (ResNet-50) get positive
    running variances and an int64 scalar num_batches_tracked, so the reference loads them with strict=True."""
    sd = OrderedDict()
    for name, shape in param_shapes(cfg_name).items():
        g = _gen(name, seed)
        n = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
        if name.endswith("sizes_of_interest"):
            t = torch.tensor([64.0, 128.0, 256.0, 512.0, 1024.0])  # dynamic_mask_head.py:106-107
        elif name.endswith("_iter"):
            t = torch.zeros(1)
        elif name.endswith("num_batches_tracked"):
            sd[name] = torch.tensor(0, dtype=torch.int64)
            continue
        elif name.endswith("running_mean"):
            t = 0.1 * n(*shape)
        elif name.endswith("running_var"):  # the stem conv sees 0-255 pixels: its BatchNorm statistics bring them to O(1)
            t = (0.5 + torch.rand(*shape, generator=g)) * (2e4 if name == "backbone.backbone.bn1.running_var" else 1.0)
        elif name.endswith("bn3.weight"):  # small residual-branch scale: activations stay O(1) through 16 un-normalised blocks
            t = 0.3 * (1.0 + 0.2 * n(*shape))
        elif name.endswith("gamma"):
            t = 0.3 * (1.0 + 0.2 * n(*shape))
        elif "beta_" in name:
            t = 1.0 + 0.2 * n(*shape)
        elif "_embed.weight" in name:
            t = torch.rand(*shape, generator=g)
        elif name.endswith("level_embed"):
            t = n(*shape)
        elif name.endswith("sampling_offsets.bias"):  # ms_deform_attn.py:64-70 grid init
            th = torch.arange(8, dtype=torch.float32) * (2.0 * math.pi / 8)
            gi = torch.stack([th.cos(), th.sin()], -1)
            gi = (gi / gi.abs().max(-1, keepdim=True)[0]).view(8, 1, 1, 2).repeat(1, 2, 4, 1)
            for i in range(4):
                gi[:, :, i, :] *= i + 1
            t = gi.reshape(-1) + 0.1 * n(*shape)
        elif name.endswith("sampling_offsets.weight"):
            t = n(*shape) * (0.5 / 16.0)
        elif name.endswith(".bias"):
            if any(k in name for k in ("obj_preds", "cls_preds")):
                t = -4.0 + 1.5 * n(*shape)
            elif "reg_preds" in name:  # wider boxes so that NMS has real work
                t = 0.1 * n(*shape) + torch.tensor([0.0, 0.0, 1.2, 1.2])
            elif any(k in name for k in (".bn.", "norm", "refine", "tower")) and len(shape) == 1 and ".0.weight" not in name:
                t = 0.1 * n(*shape)
            else:
                t = 0.1 * n(*shape)
        elif len(shape) == 1:  # norm scale
            t = 1.0 + 0.1 * n(*shape)
        else:
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            t = n(*shape) / math.sqrt(fan_in)
        sd[name] = t.float().contiguous()
    return sd


def fold_bn(w, sd, p, eps=1e-3):
    """Eval-mode BatchNorm `p` (running statistics; eps 1e-3 as init_yolo sets it, exp/unicorn_track.py:118-122) folded into the
    preceding bias-free conv weight w [Cout, ...]: s = gamma / sqrt(running_var + eps), W' = W s, b' = beta - running_mean s.
    Computed in the dtype of w."""
    s = sd[p + "weight"].to(w) / torch.sqrt(sd[p + "running_var"].to(w) + eps)
    return w * s.view(-1, *([1] * (w.dim() - 1))), sd[p + "bias"].to(w) - sd[p + "running_mean"].to(w) * s


def check_state_dict(state_dict, cfg_name, strict=True):
    """Compare a reference state_dict with the parameter table of `cfg_name`.  Returns (missing, unexpected, mismatched);
    strict=True raises a ValueError that lists them (the engine would otherwise fail later with a KeyError deep inside
    the weight packing).  Buffers the engine does not read (`head.mask_head.*`, BatchNorm `num_batches_tracked`) are ignored."""
    ignore = ("head.mask_head.", "num_batches_tracked")
    want = {k: v for k, v in param_shapes(cfg_name).items() if not any(s in k for s in ignore)}
    have = {k: tuple(v.shape) for k, v in state_dict.items() if not any(s in k for s in ignore)}
    missing = [k for k in want if k not in have]
    unexpected = [k for k in have if k not in want]
    mismatched = [(k, have[k], tuple(want[k])) for k in want if k in have and have[k] != tuple(want[k])]
    if strict and (missing or unexpected or mismatched):
        raise ValueError(f"state_dict does not match {cfg_name}: {len(missing)} missing (e.g. {missing[:3]}), "
                         f"{len(unexpected)} unexpected (e.g. {unexpected[:3]}), {len(mismatched)} shape mismatches (e.g. {mismatched[:3]})")
    return missing, unexpected, mismatched


def load_checkpoint(path_or_obj, cfg_name, strict=True):
    """The reference's checkpoint format (tools/track.py / unicorn/core/launch: torch.save({"model": state_dict, ...})): accepts the
    file path or the loaded object, a bare state_dict, and DistributedDataParallel's `module.` prefix; returns an fp32 CPU
    state_dict validated against the model's parameter table (ready for UnicornEngine / UnicornB200Model)."""
    obj = torch.load(path_or_obj, map_location="cpu", weights_only=False) if isinstance(path_or_obj, (str, bytes)) or hasattr(path_or_obj, "read") else path_or_obj
    sd = obj["model"] if isinstance(obj, dict) and "model" in obj and isinstance(obj["model"], dict) else obj
    out = OrderedDict()
    for k, v in sd.items():
        if not torch.is_tensor(v):
            continue
        out[k[7:] if k.startswith("module.") else k] = v.detach().to("cpu", torch.float32) if v.is_floating_point() else v.detach().cpu()
    check_state_dict(out, cfg_name, strict=strict)
    return out

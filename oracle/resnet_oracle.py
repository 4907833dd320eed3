"""CPU oracle for the ResNet-50 tracking models (exps/default/unicorn_track_r50*.py) — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A plain fp32 PyTorch restatement of the reference's ResNet-50 backbone (unicorn/models/backbone/resnet.py) over a reference-format
state_dict.  Everything after the backbone (PAFPN, interaction, embedding, correlation, heads, mask branch, post-processing) is the
ConvNeXt oracle's (oracle/unicorn_oracle.py), unchanged: only the channel widths differ.  Pinned against the UNMODIFIED reference by
tests/golden/make_golden_r50.py (golden fixtures sot_r50_320.npz, whole_r50_mask_320.npz).
"""
import torch
import torch.nn.functional as F

import unicorn_oracle as orc

# exps/default/unicorn_track_r50*.py: backbone_name "resnet50", in_channels [512, 1024, 2048]
CONFIGS = {
    "unicorn_track_r50": dict(backbone="resnet50", depths=(3, 4, 6, 3), num_classes=8, mask=False),
    "unicorn_track_r50_mask": dict(backbone="resnet50", depths=(3, 4, 6, 3), num_classes=8, mask=True),
}


def batchnorm_eval(x, sd, p, eps=1e-3):
    """BatchNorm2d in eval mode with the running statistics; eps 1e-3 from init_yolo (exp/unicorn_track.py:118-122,145)."""
    return F.batch_norm(x, sd[p + "running_mean"], sd[p + "running_var"], sd[p + "weight"], sd[p + "bias"], False, 0.0, eps)


def resnet50_features(img, sd, cfg, p="backbone.backbone."):
    """ResNet._forward_impl — backbone/resnet.py:206-224 (out_indices [1,2,3]); Bottleneck.forward :104-124 (v1.5: the stride
    sits on conv2; downsample = conv1x1(stride) + BN in block 0 of every layer; ReLU after the residual add)."""
    x = F.relu(batchnorm_eval(F.conv2d(img, sd[p + "conv1.weight"], stride=2, padding=3), sd, p + "bn1."))
    x = F.max_pool2d(x, 3, 2, 1)
    outs = []
    for i, n in enumerate(cfg["depths"]):
        for j in range(n):
            q = p + f"layer{i + 1}.{j}."
            s = 2 if i > 0 and j == 0 else 1
            y = F.relu(batchnorm_eval(F.conv2d(x, sd[q + "conv1.weight"]), sd, q + "bn1."))
            y = F.relu(batchnorm_eval(F.conv2d(y, sd[q + "conv2.weight"], stride=s, padding=1), sd, q + "bn2."))
            y = batchnorm_eval(F.conv2d(y, sd[q + "conv3.weight"]), sd, q + "bn3.")
            idt = batchnorm_eval(F.conv2d(x, sd[q + "downsample.0.weight"], stride=s), sd, q + "downsample.1.") if j == 0 else x
            x = F.relu(y + idt)
        if i >= 1:
            outs.append(x)
    return outs  # [s8, s16, s32]


def forward_backbone(img, sd, cfg):
    """Unicorn.forward_backbone — unicorn.py:231-258 with the ResNet-50 features.  Returns (fpn_outs, seq_dict)."""
    feats = resnet50_features(img, sd, cfg)
    fpn = orc.pafpn(feats, sd)
    feat = feats[1]
    h, w = feat.shape[-2:]
    return fpn, {"feat": feat, "pos": orc.pos_embed(sd, h, w), "h": h, "w": w}


def whole_forward(img, sd, cfg):
    """Unicorn.forward(mode="whole") — unicorn.py:133-139, as unicorn_oracle.whole_forward."""
    fpn, seq = forward_backbone(img, sd, cfg)
    bs, _, H, W = img.shape
    zeros = tuple(torch.zeros(bs, 1, H // s, W // s) for s in orc.STRIDES)
    if cfg["mask"]:
        return orc.head_forward_mask(fpn, zeros, sd, cfg, "mot"), seq
    return orc.head_forward(fpn, zeros, sd, cfg, "mot"), seq


class SOTOracle:
    """UnicornSOTTrack.initialize/track (external/lib/test/tracker/unicorn_sot.py:39-109) with the ResNet-50 backbone."""

    def __init__(self, sd, cfg_name, conf=0.001, nms=0.65, half_corr=False):
        self.sd, self.cfg = sd, CONFIGS[cfg_name]
        self.conf, self.nms, self.half_corr = conf, nms, half_corr

    @torch.no_grad()
    def initialize(self, ref_frame, init_box_xyxy):
        _, self.pre = forward_backbone(ref_frame, self.sd, self.cfg)
        H, W = ref_frame.shape[-2:]
        self.dh, self.dw = self.pre["h"] * 2, self.pre["w"] * 2
        self.lbs_pre = orc.label_map_s8(init_box_xyxy, H, W)

    @torch.no_grad()
    def track(self, cur_frame, stages=None):
        fpn, cur = forward_backbone(cur_frame, self.sd, self.cfg)
        f_pre, f_cur = orc.deform_interaction(self.pre, cur, self.sd)
        e_pre, e_cur = orc.upsample_embed(f_pre, self.sd), orc.upsample_embed(f_cur, self.sd)
        pred = orc.corr_propagate(e_pre.flatten(-2)[0], e_cur.flatten(-2)[0], self.lbs_pre, half=self.half_corr)
        coarse = pred.view(1, -1, self.dh, self.dw)
        out = orc.head_forward(fpn, orc.prior_pyramid(coarse), self.sd, self.cfg, "sot")
        dets = orc.postprocess(out, 1, self.conf, self.nms)[0]
        if stages is not None:
            stages.update(fpn=fpn, feat=cur["feat"], pos=cur["pos"], inter_pre=f_pre, inter_cur=f_cur, embed_pre=e_pre,
                          embed_cur=e_cur, coarse=coarse, head=out, dets=dets)
        return dets

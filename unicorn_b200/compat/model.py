"""Reference-shaped facade over UnicornEngine: the call conventions the reference's drivers use on `Unicorn`
(unicorn/models/unicorn.py:60-139; SURVEY.md 8b "Python model API to keep"), with the reference's tensor formats at the
boundary (NCHW fp32 in, NCHW fp32 out) so that `unicorn_sot.py` / `unicorn_vos.py` / `mot_evaluator.py`-style code runs on the H100
path unchanged:

    model = get_exp("exps/default/unicorn_track_large", None).get_model(load_pretrain=False)   # unicorn_b200/shim/unicorn/exp
    model.load_state_dict(ckpt["model"]); model.cuda(); model.eval()
    fpn_outs, seq_dict = model(imgs=x, mode="backbone")                         # unicorn.py:97-101
    f0, f1 = model(seq_dict0=a, seq_dict1=b, mode="interaction")               # unicorn.py:102-110
    emb = model(feat=f1, mode="upsample")                                      # unicorn.py:111-113
    out, seq_dict = model(imgs=x, mode="whole")                                # unicorn.py:133-139
    out = model.head(fpn_outs, prior_pyramid, mode="sot" | "mot")             # unicorn_head.py:249-336; mask models return
                                                                               # UnicornHeadMask's 6-tuple (unicorn_head_mask.py:451-471)
    dets = postprocess(out, num_classes, conf_thre, nms_thre)                  # utils/boxes.py:33-77
    dets, masks = postprocess_inst(out, locations, dyn, levels, mask_feats, model.head.mask_head, ncls, conf, nms, d_rate=2,
                                   up_masks=up_masks)                          # utils/boxes.py:80-152

Inside, everything runs on the engine's NHWC bf16 kernels; the conversions at the boundary are exact in the outbound
direction (bf16 -> fp32) and in the inbound direction for tensors that came out of this facade (their fp32 values are bf16
numbers).  `seq_dict` holds plain tensors (keys feat, pos, h, w) and survives copy.deepcopy (mot_evaluator.py:1015).  The
fused fast paths (correlation without the N x N matrix, CUDA-graph frames) live in the driver classes
(unicorn_b200.sot / mot / vos / mots), which is where a per-frame loop should go; this class is the drop-in for code that calls
the model stage by stage.  There is no CPU path: the engine is built by `.cuda()` / `.to("cuda")` (or by the constructor when a
state_dict is given) and raises without an sm_90 GPU; tensors must be CUDA tensors on the engine's device."""
import collections
import math

import torch

from .. import ops, post_ops
from ..engine import UnicornEngine
from ..weights import CONFIGS, param_shapes

_IncompatibleKeys = collections.namedtuple("IncompatibleKeys", ["missing_keys", "unexpected_keys"])
STRIDES = (8, 16, 32)


def _nhwc(x):
    assert x.is_cuda and x.dim() == 4, "UnicornB200Model: CUDA NCHW tensors only (no CPU fallback)"
    return ops.nchw_to_nhwc(x.float().contiguous())


class _MaskHeadHandle:
    """What `model.head.mask_head` is passed around for (utils/boxes.py:80, dynamic_mask_head.py): postprocess_inst of this
    package runs the dynamic-conv mask head as CUDA kernels and only needs the constants."""
    soi = (64.0, 128.0, 256.0)


class _Head:
    def __init__(self, model):
        self._m = model
        self.decode_in_inference = True
        self.mask_head = _MaskHeadHandle() if model.cfg["mask"] else None

    def __call__(self, fpn_outs, prior_ms=None, mode="sot"):
        """fpn_outs: 3 NCHW fp32 maps (B,C,h,w); prior_ms: 3 fp32 maps (B,1,h,w).  -> (B, A, 5+ncls), or (B = 1 only)
        UnicornHeadMask's tuple (outputs, locations (A,2), dynamic_params (1,A,169), fpn_levels (1,A), mask_feats (1,8,h,w),
        up_masks (1,144,h,w))."""
        e = self._m._engine()
        B = fpn_outs[0].shape[0]
        if self._m.cfg["mask"] and B != 1:
            raise ValueError(f"UnicornB200Model.head: the mask head runs one image per call (got a batch of {B})")
        fpn = [_nhwc(t) for t in fpn_outs]
        pri = None
        if prior_ms is not None:
            if mode == "sot":
                pri = [p.float().reshape(B, p.shape[-2], p.shape[-1]).contiguous() for p in prior_ms]
            else:  # the reference adds x + m * beta in "mot" mode too; its only caller passes zeros (unicorn.py:136-139)
                assert all(float(p.abs().max()) == 0.0 for p in prior_ms), "non-zero priors with mode='mot' are not supported"
        e.begin_frame()
        mask = self._m.cfg["mask"]
        out = e.head(fpn, pri, mode, with_masks=mask).clone()
        if not mask:
            return out
        dyn = torch.cat([d[0, :, :, :169].reshape(-1, 169) for d in e.dyn_levels], 0)[None].contiguous()
        locs, lvls = [], []
        for k, d in enumerate(e.dyn_levels):
            h, w = d.shape[1:3]
            yv, xv = torch.meshgrid(torch.arange(h, device=d.device), torch.arange(w, device=d.device), indexing="ij")
            locs.append((torch.stack((xv, yv), 2).view(-1, 2).float() + 0.5) * STRIDES[k])  # unicorn_head_mask.py:518
            lvls.append(torch.full((1, h * w), k, device=d.device, dtype=torch.long))
        mf, um = e.mask_branch(fpn)
        # mask-branch outputs are fp32 NHWC (ops.nhwc_to_nchw converts 16-bit maps): plain permutes at this compatibility boundary
        return out, torch.cat(locs, 0), dyn, torch.cat(lvls, 1), mf.permute(0, 3, 1, 2).contiguous(), um.permute(0, 3, 1, 2).contiguous()


class UnicornB200Model:
    def __init__(self, state_dict=None, cfg_name="unicorn_track_large", device="cuda"):
        assert cfg_name in CONFIGS, f"unknown config {cfg_name!r} (known: {sorted(CONFIGS)})"
        self.cfg_name, self.cfg = cfg_name, CONFIGS[cfg_name]
        self.num_classes = self.cfg["num_classes"]
        self._sd = None
        self._device = device
        self.engine = None
        self._on_gpu = False
        self.training = False
        self.head = _Head(self)
        if state_dict is not None:
            self.load_state_dict(state_dict)
            self.cuda(device)

    # ---- nn.Module-shaped life cycle (exp/unicorn_track.py:115-193; unicorn_sot.py:26-31; tools/track_omni.py:168-201)
    def load_state_dict(self, state_dict, strict=True):
        want = param_shapes(self.cfg_name)
        sd = {k: v for k, v in state_dict.items() if torch.is_tensor(v)}
        missing = [k for k in want if k not in sd]
        unexpected = [k for k in sd if k not in want and not k.startswith("head.mask_head.")]  # buffers of DynamicMaskHead
        for k, shp in want.items():
            if k in sd and tuple(sd[k].shape) != tuple(shp):
                raise RuntimeError(f"size mismatch for {k}: checkpoint {tuple(sd[k].shape)}, model {tuple(shp)}")
        if strict and (missing or unexpected):
            raise RuntimeError(f"Error(s) in loading state_dict for UnicornB200Model: missing key(s) {missing[:8]}, unexpected key(s) {unexpected[:8]}")
        if missing:  # strict=False (tools/track_omni.py:196) tolerates extra keys; the engine still needs every inference parameter
            raise RuntimeError(f"UnicornB200Model needs every inference parameter; missing {missing[:8]}{'...' if len(missing) > 8 else ''}")
        self._sd = sd
        if self._on_gpu:  # .cuda() came first (tools/track_omni.py:170,196) or the weights are being replaced: (re)build
            self.engine = UnicornEngine(self._sd, self.cfg_name, device=self._device)
        return _IncompatibleKeys(missing, unexpected)

    def cuda(self, device=None):
        if device is not None:
            self._device = device if not isinstance(device, int) else f"cuda:{device}"
        self._on_gpu = True
        if self.engine is None and self._sd is not None:
            self.engine = UnicornEngine(self._sd, self.cfg_name, device=self._device)  # raises without an sm_90 GPU: no CPU fallback
        return self

    def to(self, device=None, *a, **k):
        if device is not None and str(device).startswith("cuda"):
            return self.cuda(device)
        if device is not None and str(device) == "cpu":
            raise RuntimeError("UnicornB200Model has no CPU path")
        return self

    def eval(self):
        self.training = False
        return self

    def train(self, mode=True):
        if mode:
            raise RuntimeError("UnicornB200Model is inference only (training is out of scope, SURVEY.md section 8)")
        return self

    def half(self):  # the reference's --fp16 switch: the engine already computes in bf16 / fp16
        return self

    def float(self):
        return self

    def _engine(self):
        if self.engine is None:
            raise RuntimeError("UnicornB200Model: needs load_state_dict(...) and .cuda() before the first call (GPU only, no default weights)")
        return self.engine

    def _backbone(self, imgs):
        e = self._engine()
        assert imgs.is_cuda and imgs.dim() == 4 and imgs.shape[0] >= 1, "CUDA NCHW frames [B,3,H,W]"
        e.begin_frame()
        fpn, seq = e.backbone(imgs.float().contiguous(), tag="compat")
        h, w = seq["h"], seq["w"]
        seq_dict = {"feat": ops.nhwc_to_nchw(seq["feat"]), "pos": e.pos_tokens(h, w)[1].clone(), "h": h, "w": w}
        return fpn, seq_dict

    def __call__(self, imgs=None, seq_dict0=None, seq_dict1=None, feat=None, mode="backbone", **unused):
        e = self._engine()
        if self.cfg["task"] == "det":  # YOLOX.forward (models/yolox.py:28-50): NCHW fp32 [B,3,H,W] -> decoded [B, A, 5+ncls]
            if not self.head.decode_in_inference:
                raise ValueError("UnicornB200Model: the detector returns decoded outputs only (head.decode_in_inference=True)")
            assert imgs.is_cuda and imgs.dim() == 4 and imgs.shape[0] >= 1, "CUDA NCHW images [B,3,H,W]"
            e.begin_frame()
            fpn, _ = e.backbone(imgs.float().contiguous(), tag="compat")
            if not self.cfg["mask"]:
                return e.head(fpn, None, "mot").clone()
            # YOLOXHeadDetMask (yolo_head_det_mask.py:344-363, use_raft): (decoded [B,A,85], locations [A,2], dynamic_params [B,A,169],
            # fpn_levels [B,A], mask_feats [B,8,h,w], up_masks [B,144,h,w])
            out = e.head(fpn, None, "mot", with_masks=True).clone()
            B = out.shape[0]
            dyn = torch.cat([d[..., :169].reshape(B, -1, 169) for d in e.dyn_levels], 1).contiguous()
            locs, lvls = [], []
            for k, d in enumerate(e.dyn_levels):
                h, w = d.shape[1:3]
                yv, xv = torch.meshgrid(torch.arange(h, device=d.device), torch.arange(w, device=d.device), indexing="ij")
                locs.append((torch.stack((xv, yv), 2).view(-1, 2).float() + 0.5) * STRIDES[k])  # decode_outputs :404
                lvls.append(torch.full((B, h * w), k, device=d.device, dtype=torch.long))
            mf, um = e.mask_branch(fpn)
            return out, torch.cat(locs, 0), dyn, torch.cat(lvls, 1), mf.permute(0, 3, 1, 2).contiguous(), um.permute(0, 3, 1, 2).contiguous()
        if mode == "backbone":
            fpn, seq_dict = self._backbone(imgs)
            return tuple(ops.nhwc_to_nchw(t) for t in fpn), seq_dict
        if mode == "interaction":
            e.begin_frame()
            f0, f1 = e.interaction(_nhwc(seq_dict0["feat"]), _nhwc(seq_dict1["feat"]))
            return ops.nhwc_to_nchw(f0), ops.nhwc_to_nchw(f1)
        if mode == "upsample":
            return ops.nhwc_to_nchw(e.upsample(_nhwc(feat), "compat"))
        if mode == "whole":  # backbone + head with zero priors, MOT prediction set (unicorn.py:133-139)
            if self.cfg["mask"] and imgs.shape[0] != 1:
                raise ValueError(f"UnicornB200Model(mode='whole'): the mask head runs one image per call (got a batch of {imgs.shape[0]})")
            fpn, seq_dict = self._backbone(imgs)
            if not self.cfg["mask"]:
                return e.head(fpn, None, "mot").clone(), seq_dict
            return self.head(tuple(ops.nhwc_to_nchw(t) for t in fpn), None, mode="mot"), seq_dict
        raise ValueError(f"UnicornB200Model: unsupported mode {mode!r} (inference modes: backbone, interaction, upsample, whole)")


def _to_corners_(prediction):
    """utils/boxes.py:34-39 — the reference converts cxcywh to corners IN PLACE on the caller's tensor; kept for drop-in parity."""
    c = prediction.new_empty(prediction.shape[:-1] + (4,))
    c[..., 0] = prediction[..., 0] - prediction[..., 2] / 2
    c[..., 1] = prediction[..., 1] - prediction[..., 3] / 2
    c[..., 2] = prediction[..., 0] + prediction[..., 2] / 2
    c[..., 3] = prediction[..., 1] + prediction[..., 3] / 2
    prediction[..., :4] = c


def postprocess(prediction, num_classes, conf_thre=0.7, nms_thre=0.45, class_agnostic=False):
    """unicorn.utils.postprocess (utils/boxes.py:33-77): list with one (M,7) tensor of rows per image
    (x1,y1,x2,y2,obj_conf,class_conf,class_pred), descending score, or None when nothing passes — on the GPU, every image of the
    batch in one launch sequence.  Like the reference, the boxes of `prediction` are converted to corner form in place.
    class_agnostic=True: NMS across classes (torchvision.ops.nms, as tools/demo.py asks for)."""
    p = prediction.float().contiguous()
    B, A = p.shape[:2]
    ws = ops.PostWorkspace(A, p.device, B)
    if class_agnostic:
        dets, cnt = post_ops.postprocess_device_ex(p, num_classes, conf_thre, nms_thre, ws, class_agnostic=True)
    else:
        dets, cnt = ops.postprocess_device(p, num_classes, conf_thre, nms_thre, ws)
    dets = dets.view(B, A, 7)
    out = [dets[i, :n].clone() if n > 0 else None for i, n in enumerate(cnt.tolist())]
    _to_corners_(prediction)
    return out


def postprocess_inst(prediction, locations, dynamic_params, fpn_levels, mask_feats, mask_head, num_classes, conf_thre=0.7, nms_thre=0.45,
                     class_agnostic=False, d_rate=4, up_masks=None):
    """unicorn.utils.boxes.postprocess_inst (utils/boxes.py:80-152): (list of (M,7) detections, list of (M,1,H,W) sigmoid masks).
    `locations` / `fpn_levels` are implied by the anchor order (level-major, row-major) and only checked for size; `mask_head` is
    the handle returned as model.head.mask_head."""
    if class_agnostic:
        raise NotImplementedError("postprocess_inst(class_agnostic=True): the tracking drivers use class-aware NMS (unicorn_vos.py:191)")
    if up_masks is None:
        raise NotImplementedError("postprocess_inst without up_masks (use_raft=False): the released tracking models use the RAFT upsampler")
    bs, A, _ = prediction.shape
    _, _, h, w = mask_feats.shape
    hw = [(h, w), (h // 2, w // 2), (h // 4, w // 4)]
    assert sum(a * b for a, b in hw) == A == dynamic_params.shape[1] == locations.shape[0]
    up_rate = int(round(math.sqrt(up_masks.shape[1] / 9)))
    outs, out_masks = [], []
    for i in range(bs):
        p = prediction[i].float().contiguous()
        ws = ops.PostWorkspace(A, p.device)
        dets, cnt = ops.postprocess_device(p, num_classes, conf_thre, nms_thre, ws)
        n = int(cnt.item())
        if n == 0:
            outs.append(None)
            out_masks.append(None)
            continue
        dyn = dynamic_params[i].float().contiguous()
        levels, off = [], 0
        for a, b in hw:
            levels.append(dyn[off:off + a * b].view(1, a, b, 169))
            off += a * b
        mf = mask_feats[i:i + 1].float().permute(0, 2, 3, 1).contiguous()
        um = (up_masks[0:1] if len(up_masks) == 1 else up_masks[i:i + 1]).float().permute(0, 2, 3, 1).contiguous()
        masks = ops.dynamic_masks(mf, um, levels, hw, ws, n, up_rate=up_rate, d_rate=d_rate, soi=_MaskHeadHandle.soi)
        outs.append(dets[:n].clone())
        out_masks.append(masks[:, None])
    _to_corners_(prediction)
    return outs, out_masks

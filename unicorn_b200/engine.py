"""UnicornEngine — the per-frame inference hot path as a static sequence of sm_90a kernel launches.

Host-side mirror of the reference model (unicorn/models/unicorn.py `Unicorn`, backbone/yolo_pafpn_new.py,
backbone/convnext.py, deformable_transformer.py, unicorn_head.py) with an H100-first data layout:

  * activations live in HBM as NHWC bf16 (channels contiguous): LayerNorm/Linear of ConvNeXt need no permutes and
    every convolution is an implicit GEMM whose A operand is fetched by TMA boxes straight from the NHWC map;
  * concatenations (PAFPN, CSP) are never materialised by copies: producers write into channel slices of one buffer;
  * GroupNorm statistics are accumulated in the producing convolution's epilogue, the normalise+SiLU pass runs in place;
  * the embedding used for correlation is written as fp16 (the reference casts to .half() before torch.mm);
  * prediction logits, statistics, priors and boxes stay fp32.

All buffers are allocated on first use per input resolution and then reused, so a steady-state frame performs no
allocation and can be captured in a CUDA graph (see unicorn_b200/sot.py).  torch is used only as the device-memory
allocator and stream/graph plumbing; every arithmetic step is a launch through the C ABI (unicorn_b200/ops.py).
"""
import os

import torch

from . import ops, shared_ops
from .weights import CONFIGS, fold_bn

ACT_NONE, ACT_RELU, ACT_GELU, ACT_SILU = ops.ACT_NONE, ops.ACT_RELU, ops.ACT_GELU, ops.ACT_SILU
BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
STRIDES = (8, 16, 32)


class _ConvGN:
    """BaseConv: conv (no bias) -> GroupNorm -> SiLU (network_blocks.py:29-51, GN via exp/unicorn_track.py:450-470)."""

    def __init__(self, w, gw, gb, k, stride, groups=16, eps=1e-3, bias=None):
        self.w, self.gw, self.gb, self.k, self.stride, self.groups, self.eps, self.bias = w, gw, gb, k, stride, groups, eps, bias
        self.cout = w.shape[0]


class UnicornEngine:
    def __init__(self, state_dict, cfg_name, device="cuda", autotune=True, ln_fold=False):
        ops._lib.check(ops._lib.lib().uc_check_device(), "uc_check_device")  # fail loudly without an sm_90 GPU
        self.cfg_name = cfg_name
        self.cfg = CONFIGS[cfg_name]
        self.dev = torch.device(device)
        self.dims = self.cfg["dims"]
        self.inc = self.cfg["in_channels"]  # channels of the s8 / s16 / s32 backbone outputs
        self.depths = self.cfg["depths"]
        self.ncls = self.cfg["num_classes"]
        self._bufs = {}
        self._stats_arena = None
        self._stats_used = 0
        self._retired = []
        self._pos_cache = {}
        self._side_streams = None
        self._fork_stream = None
        self._with_masks = False
        self._bn_cache = {}
        self._bn_dirty = False
        # ln_fold: the LayerNorm of the ConvNeXt blocks without a fused MLP is folded into pwconv1 (statistics from the fp32-FMA
        # depthwise kernel, normalisation in the GEMM epilogue; tests/test_lnfold_gpu.py); off by default
        self.ln_fold = bool(ln_fold)
        self._row_arena, self._row_used = None, 0
        self._ctr_arena, self._ctr_used = None, 0  # work counters of the dynamically scheduled kernels (zeroed by begin_frame)
        self.autotune = autotune
        self.load_tuning()
        self._load(state_dict)

    def fork(self):
        """A second execution context on the SAME weights: its own activation buffers, statistics arenas and side streams, so that
        two frames can be in flight on two streams (frames of a video are independent until association; see sot.py submit /
        collect).  Packed weights, position tables and the tuning table are shared."""
        import copy
        ctx = copy.copy(self)
        ctx._bufs = {}
        ctx._stats_arena, ctx._stats_used, ctx._retired = None, 0, []
        ctx._row_arena, ctx._row_used = None, 0
        ctx._ctr_arena, ctx._ctr_used = None, 0
        ctx._side_streams, ctx._fork_stream = None, None
        return ctx

    def _tracking_only(self, what):
        if self.det:
            raise ValueError(f"UnicornEngine.{what}: {self.cfg_name} is a detector (backbone, neck and head only); "
                             f"{what} belongs to the tracking models")

    # ------------------------------------------------------------------------------------------ weights
    def _load(self, sd):
        dev = self.dev
        f = lambda k: sd[k].to(dev, F32).contiguous()  # noqa: E731
        pw = lambda k: ops.pack_conv_weight(sd[k].to(dev, F32))  # noqa: E731
        P = {}
        b = "backbone.backbone."

        def block(p):
            d = dict(dw=ops.pack_dw_weight(sd[p + "dwconv.weight"].to(dev)), dwm=ops.pack_dw_weight_mma(sd[p + "dwconv.weight"].to(dev), sd[p + "dwconv.bias"].to(dev)), dwb=f(p + "dwconv.bias"), lnw=f(p + "norm.weight"),
                     lnb=f(p + "norm.bias"), w1=pw(p + "pwconv1.weight"), b1=f(p + "pwconv1.bias"), w2=pw(p + "pwconv2.weight"),
                     b2=f(p + "pwconv2.bias"), gamma=f(p + "gamma"))
            # LayerNorm -> pwconv1 -> GELU -> pwconv2 -> layer scale -> residual in one launch for C = 96 / 192 / 256 / 384 (csrc/mlp_fused.cu)
            d["fused"] = ops.convnext_mlp_supported(d["lnw"].numel())
            if self.ln_fold or d["fused"]:  # W' = W diag(g) (16-bit), colsum(W') of the ROUNDED weights, c = W beta + b
                w1 = sd[p + "pwconv1.weight"].to(dev, F32).reshape(d["b1"].numel(), -1)
                d["w1f"] = ops.pack_conv_weight((w1 * d["lnw"][None, :])[:, :, None, None])
                d["s1"] = d["w1f"].float().sum(dim=(1, 2)).contiguous()
                d["c1"] = (w1 @ d["lnb"] + d["b1"]).contiguous()
            return d

        if self.cfg["backbone"] == "resnet50":
            self._load_resnet(sd, P, b)
        else:
            self._load_convnext(sd, P, b, f, pw, block)

        def cgn(p, k, stride=1):
            return _ConvGN(pw(p + "conv.weight"), f(p + "bn.weight"), f(p + "bn.bias"), k, stride)

        def csp(p):
            c1, c2 = cgn(p + "conv1.", 1), cgn(p + "conv2.", 1)
            fused = _ConvGN(torch.cat([c1.w, c2.w], 0).contiguous(), torch.cat([c1.gw, c2.gw]).contiguous(),
                            torch.cat([c1.gb, c2.gb]).contiguous(), 1, 1, groups=32)
            return dict(c12=fused, c3=cgn(p + "conv3.", 1), m=[(cgn(p + f"m.{i}.conv1.", 1), cgn(p + f"m.{i}.conv2.", 3)) for i in range(3)])

        n = "backbone."
        P["lateral_conv0"], P["reduce_conv1"] = cgn(n + "lateral_conv0.", 1), cgn(n + "reduce_conv1.", 1)
        P["bu_conv2"], P["bu_conv1"] = cgn(n + "bu_conv2.", 3, 2), cgn(n + "bu_conv1.", 3, 2)
        for name in ("C3_p4", "C3_p3", "C3_n3", "C3_n4"):
            P[name] = csp(n + name + ".")
        self.det = self.cfg["task"] == "det"
        if not self.det:  # a detector (YOLOX) has no interaction, upsampling or SOT predictors
            self._load_interaction(sd, P, f, pw)
        # head
        self._load_head(sd, P, f, pw, cgn, block)
        self.P = P

    def _load_interaction(self, sd, P, f, pw):
        dev = self.dev
        P["bottleneck"] = _ConvGN(pw("bottleneck.0.weight"), f("bottleneck.1.weight"), f("bottleneck.1.bias"), 1, 1, groups=32, eps=1e-5,
                                  bias=f("bottleneck.0.bias"))
        t = "transformer.encoder.layers.0."
        P["value_proj"] = (pw(t + "self_attn.value_proj.weight"), f(t + "self_attn.value_proj.bias"))
        P["offlog"] = (ops.pack_conv_weight(torch.cat([sd[t + "self_attn.sampling_offsets.weight"], sd[t + "self_attn.attention_weights.weight"]], 0).to(dev, F32)),
                       torch.cat([sd[t + "self_attn.sampling_offsets.bias"], sd[t + "self_attn.attention_weights.bias"]]).to(dev, F32).contiguous())
        P["output_proj"] = (pw(t + "self_attn.output_proj.weight"), f(t + "self_attn.output_proj.bias"))
        P["norm1"] = (f(t + "norm1.weight"), f(t + "norm1.bias"))
        P["linear1"] = (pw(t + "linear1.weight"), f(t + "linear1.bias"))
        P["linear2"] = (pw(t + "linear2.weight"), f(t + "linear2.bias"))
        P["norm2"] = (f(t + "norm2.weight"), f(t + "norm2.bias"))
        P["level_embed"] = f("transformer.level_embed")
        P["pos_tab"] = (f("pos_emb.col_embed.weight"), f("pos_emb.row_embed.weight"))
        P["up1"] = (pw("upsample_layer.1.weight"), f("upsample_layer.1.bias"))
        P["up3"] = (pw("upsample_layer.3.weight"), f("upsample_layer.3.bias"))

    def _load_head(self, sd, P, f, pw, cgn, block):
        dev = self.dev
        h = "head."
        P["head"] = []
        for k in range(3):
            lvl = dict(stem=cgn(h + f"stems.{k}.", 1), beta=None if self.det else f(h + f"beta_{k}").reshape(-1).contiguous(),
                       att=[block(h + f"att_layers.{k}.{i}.") for i in range(3)],
                       cls=[cgn(h + f"cls_convs.{k}.{i}.", 3) for i in range(4)], reg=[cgn(h + f"reg_convs.{k}.{i}.", 3) for i in range(4)])
            for sfx in ("",) if self.det else ("", "_sot"):
                ro_w = torch.cat([sd[h + f"reg_preds{sfx}.{k}.weight"], sd[h + f"obj_preds{sfx}.{k}.weight"]], 0).to(dev, F32)
                ro_b = torch.zeros(8, device=dev)
                ro_b[:5] = torch.cat([sd[h + f"reg_preds{sfx}.{k}.bias"], sd[h + f"obj_preds{sfx}.{k}.bias"]]).to(dev)
                cw = sd[h + f"cls_preds{sfx}.{k}.weight"].to(dev, F32)
                cb = torch.zeros(_cls_cols(cw.shape[0]), device=dev)  # bias of the packed (8-row padded) class conv
                cb[:cw.shape[0]] = sd[h + f"cls_preds{sfx}.{k}.bias"].to(dev)
                lvl["pred" + sfx] = (ops.pack_conv_weight(ro_w), ro_b, ops.pack_conv_weight(cw), cb, cw.shape[0])
            if self.cfg["mask"]:  # controller conv3x3 256 -> 169 dynamic-conv parameters (unicorn_head_mask.py:238-247,333-334)
                cb = torch.zeros(176, device=dev)
                cb[:169] = sd[h + f"controllers.{k}.bias"].to(dev)
                lvl["ctrl"] = (pw(h + f"controllers.{k}.weight"), cb)
            P["head"].append(lvl)
        if self.cfg["mask"]:  # MaskBranch (condinst/mask_branch.py:17-70), BN -> GN16 eps 1e-3, ReLU
            mb = h + "mask_branch."
            cgr = lambda p: _ConvGN(pw(p + "0.weight"), f(p + "1.weight"), f(p + "1.bias"), 3, 1)  # noqa: E731
            P["mask"] = dict(refine=[cgr(mb + f"refine.{k}.") for k in range(3)], tower=[cgr(mb + f"tower.{i}.") for i in range(4)],
                             out=(pw(mb + "tower.4.weight"), f(mb + "tower.4.bias")),
                             up0=(pw(mb + "up_mask_layer.0.weight"), f(mb + "up_mask_layer.0.bias")),
                             up2=(pw(mb + "up_mask_layer.2.weight"), f(mb + "up_mask_layer.2.bias")))

    def _load_convnext(self, sd, P, b, f, pw, block):
        dev = self.dev
        P["stem"] = (ops.pack_stem_weight(sd[b + "downsample_layers.0.0.weight"].to(dev)), f(b + "downsample_layers.0.0.bias"),
                     f(b + "downsample_layers.0.1.weight"), f(b + "downsample_layers.0.1.bias"))
        for i in range(1, 4):
            P[f"down{i}"] = (f(b + f"downsample_layers.{i}.0.weight"), f(b + f"downsample_layers.{i}.0.bias"),
                             pw(b + f"downsample_layers.{i}.1.weight"), f(b + f"downsample_layers.{i}.1.bias"))
            P[f"outnorm{i}"] = (f(b + f"norm{i}.weight"), f(b + f"norm{i}.bias"))
        P["stages"] = [[block(b + f"stages.{i}.{j}.") for j in range(self.depths[i])] for i in range(4)]

    def _load_resnet(self, sd, P, b):
        """ResNet-50 (backbone/resnet.py) with every eval-mode BatchNorm folded into its conv (fp32 fold, then one rounding to 16 bits)."""
        dev = self.dev
        sd = {k: v.to(dev) for k, v in sd.items() if k.startswith(b)}

        def cb(conv, bn):
            w, bias = fold_bn(sd[conv].to(F32), sd, bn)
            return ops.pack_conv_weight(w), bias.contiguous()

        w, bias = fold_bn(sd[b + "conv1.weight"].to(F32), sd, b + "bn1.")
        P["rstem"] = (ops.pack_resnet_stem_weight(w), bias.contiguous())
        P["layers"] = []
        for i, n in enumerate(self.depths):
            blocks = []
            for j in range(n):
                q = b + f"layer{i + 1}.{j}."
                d = dict(c1=cb(q + "conv1.weight", q + "bn1."), c2=cb(q + "conv2.weight", q + "bn2."), c3=cb(q + "conv3.weight", q + "bn3."),
                         stride=2 if i > 0 and j == 0 else 1)
                if j == 0:
                    d["ds"] = cb(q + "downsample.0.weight", q + "downsample.1.")
                blocks.append(d)
            P["layers"].append(blocks)

    # ------------------------------------------------------------------------------------------ buffers
    def buf(self, name, shape, dtype=BF16, zero=False):
        key = (name, tuple(shape), dtype)
        t = self._bufs.get(key)
        if t is None:
            t = (torch.zeros if zero else torch.empty)(*shape, dtype=dtype, device=self.dev)
            self._bufs[key] = t
        return t

    # ------------------------------------------------------------------------------------------ conv autotuning
    def conv(self, x, w, k, stride=1, pad=0, out=None, **kw):
        """ops.conv2d with a plan-time choice of the N tile: the first time a layer shape is seen (outside CUDA-graph
        capture) every valid block_n is timed on scratch outputs and the fastest is cached."""
        B, H, W, Cin = x.shape
        Cout = w.shape[0]
        gn = kw.get("gn_groups", 0)
        res_key = "act_after_res" if kw.get("act_after_res") else kw.get("res") is not None  # residual field: none / res + act(y) / act(y + res)
        key = (B, H, W, Cin, Cout, k, stride, pad, kw.get("act", 0), gn, res_key, out.dtype) + (("lnfold",) if kw.get("row_stats") is not None else ())
        key = "|".join(str(v) for v in key)
        bn = self._bn_cache.get(key)
        if bn is None:
            bn = 0
            if self.autotune and not torch.cuda.is_current_stream_capturing():
                bn = self._tune(x, w, k, stride, pad, out, kw, Cout, gn)
                self._bn_dirty = True
            self._bn_cache[key] = bn
        return ops.conv2d(x, w, k, k, stride, pad, out=out, block_n=bn, **kw)

    def _tune(self, x, w, k, stride, pad, out, kw, Cout, gn):
        gs = Cout // gn if gn else 0
        cands = [0] + [b for b in (64, 96, 128, 192, 256) if (not gs or b % gs == 0) and b < 2 * Cout + 64]
        cands += [1000 + b for b in (128, 192, 256) if b in cands]  # 2-CTA cluster variants with weight multicast
        scratch = torch.empty_like(out)
        kw2 = dict(kw)
        if gn:
            kw2["gn_stats"] = torch.zeros(out.shape[0], gn, 2, dtype=torch.int64, device=self.dev)
        best, best_t, times = 0, None, []
        reps = 6
        # objective: launch time discounted by the share of the SMs the launch occupies, t * (w + (1 - w) * min(CTAs, SMs) / SMs) with
        # w = UC_TUNE_SMTIME_W (default 0.5; 1 = pure latency): with several frames in flight a launch on fewer CTAs leaves SMs to the other
        # frames' kernels
        w_lat = float(os.environ.get("UC_TUNE_SMTIME_W", "0.5"))
        sms = torch.cuda.get_device_properties(self.dev).multi_processor_count
        m_tiles = -(-(out.shape[0] * out.shape[1] * out.shape[2]) // 128)
        for bn in cands:
            # timed as the frame runs it: back-to-back kernel nodes of a CUDA graph (stream launches of ~20 us kernels
            # measure launch cadence, not the kernel)
            try:
                ops.conv2d(x, w, k, k, stride, pad, out=scratch, block_n=bn, **kw2)
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    for _ in range(reps):
                        ops.conv2d(x, w, k, k, stride, pad, out=scratch, block_n=bn, **kw2)
                g.replay()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                g.replay()
                g.replay()
                e1.record()
                e1.synchronize()
                t = e0.elapsed_time(e1) / (2 * reps)
                del g
            except ops._lib.UnicornB200Error:
                continue
            times.append((bn, round(t * 1e3, 1)))  # us per launch
            if w_lat < 1.0 and bn:
                ctas = m_tiles * -(-Cout // (bn % 1000))
                t = t * (w_lat + (1.0 - w_lat) * min(ctas, sms) / sms)
            if best_t is None or t < best_t * 0.97:  # require a 3 % win to leave the earlier (heuristic-first) choice
                best, best_t = bn, t
        if os.environ.get("UC_TUNE_LOG"):
            print("tune", tuple(x.shape), "->", Cout, "k", k, "s", stride, "gn", gn, "best", best, times, flush=True)
        return best

    def tuning_path(self):
        return os.path.join(os.path.dirname(os.path.abspath(__file__)), "tuned", f"{self.cfg_name}.json")

    def load_tuning(self, path=None):
        """Per-layer N-tile choices committed under unicorn_b200/tuned/ (measured on an H100 80GB HBM3 at a 700 W power limit;
        plan-time autotuning fills in whatever is missing).
        Returns the number of entries loaded."""
        import glob
        import json
        if path is None and os.environ.get("UC_NO_TUNED"):
            return 0  # plan-time autotuning of every layer (tools: regenerate the committed tables)
        if path is None:
            # keys are layer shapes, not config names: the tables of the other configs cover the layers they share with this
            # one (e.g. *_mask and *_mot_challenge differ from unicorn_track_large only in the head outputs); this config's
            # own table is applied last
            own = self.tuning_path()
            paths = sorted(p for p in glob.glob(os.path.join(os.path.dirname(own), "*.json")) if p != own) + [own]
        else:
            paths = [path]
        for p in paths:
            if os.path.exists(p):
                self._bn_cache.update(json.load(open(p)))
        return len(self._bn_cache)

    def save_tuning(self, path):
        import json
        os.makedirs(os.path.dirname(path), exist_ok=True)
        json.dump(self._bn_cache, open(path, "w"), indent=0, sort_keys=True)

    def begin_frame(self):
        """Zero the GroupNorm statistics arena (one memset per frame; slots are handed out in call order)."""
        # every launch goes to the CURRENT device's current stream (ops._S): an engine living on another GPU must be driven under
        # torch.cuda.device(engine.dev) — one process per GPU is the intended deployment (DESIGN.md 6)
        assert self.dev.index is None or torch.cuda.current_device() == self.dev.index, \
            f"UnicornEngine on {self.dev} driven while cuda:{torch.cuda.current_device()} is current: wrap the calls in torch.cuda.device(...)"
        if self._stats_arena is None:
            self._stats_arena = torch.zeros(512, 32, 2, dtype=torch.int64, device=self.dev)
        else:
            self._stats_arena.zero_()
        self._stats_used = 0
        if self._row_arena is not None:
            self._row_arena.zero_()
        self._row_used = 0
        if self._ctr_arena is None:
            self._ctr_arena = torch.zeros(256, dtype=torch.int32, device=self.dev)
        else:
            self._ctr_arena.zero_()
        self._ctr_used = 0

    def _row_stats(self, n_pix):
        """[n_pix, 2] int64 slice of the per-frame LayerNorm-statistics arena (zeroed by begin_frame, handed out in call order)."""
        need = self._row_used + n_pix
        if self._row_arena is None or need > self._row_arena.shape[0]:
            assert not torch.cuda.is_current_stream_capturing(), "row-statistics arena must be sized by an eager frame first"
            grown = torch.zeros(max(need, 2 * (0 if self._row_arena is None else self._row_arena.shape[0]), 1 << 16), 2, dtype=torch.int64, device=self.dev)
            self._row_arena = grown  # earlier slices of this frame stay alive through the tensors that reference the old arena
        s = self._row_arena[self._row_used:need]
        self._row_used = need
        return s

    def _ctr(self):
        """One zeroed int32 work counter (uc_dwconv7 hands out its tiles with it), in call order like the statistics slots."""
        c = self._ctr_arena[self._ctr_used:self._ctr_used + 1]
        self._ctr_used += 1
        assert self._ctr_used <= self._ctr_arena.shape[0]
        return c

    def _stats(self, groups, B=1):
        """GroupNorm statistics of one conv: [G, 2] (B = 1) or [B, G, 2] int64, B consecutive slots of the per-frame arena."""
        if B == 1:
            s = self._stats_arena[self._stats_used]
            self._stats_used += 1
            assert self._stats_used <= self._stats_arena.shape[0]
            return s[:groups]
        need = self._stats_used + B
        if need > self._stats_arena.shape[0]:  # a batched frame needs B slots per conv
            assert not torch.cuda.is_current_stream_capturing(), "statistics arena must be sized by an eager frame first"
            self._retired.append(self._stats_arena)  # graphs captured earlier read and zero the old arena: it stays allocated
            self._stats_arena = torch.zeros(max(need, 2 * self._stats_arena.shape[0]), 32, 2, dtype=torch.int64, device=self.dev)
        s = self._stats_arena[self._stats_used:need]
        self._stats_used = need
        return s.view(-1)[:B * groups * 2].view(B, groups, 2)

    # ------------------------------------------------------------------------------------------ building blocks
    def conv_gn(self, x, c, out, act=ACT_SILU, prior=None, beta=None, add2=None, out2=None):
        """x NHWC view -> out NHWC view (may be a channel slice)."""
        st = self._stats(c.groups, x.shape[0])
        self.conv(x, c.w, c.k, c.stride, (c.k - 1) // 2, bias=c.bias, out=out, gn_stats=st, gn_groups=c.groups)
        ops.groupnorm_apply(out, st, c.gw, c.gb, c.groups, c.eps, act, prior=prior, beta=beta, add2=add2, out2=out2)
        return out

    def convnext_block(self, x, bp, tag):
        """In place on x (NHWC contiguous) — convnext.py:41-54."""
        B, H, W, C = x.shape
        # fused back half (csrc/mlp_fused.cu): one CTA per 128 rows.  On the head's small levels (32 and 8 row tiles at 800x1280) the launch
        # occupies few SMs but the levels run on parallel streams next to other frames in flight, so there is no size gate
        if bp["fused"]:
            t = ops.dwconv7_mma(x, bp["dwm"], out=self.buf(tag + ".t", x.shape), work_counter=self._ctr())
            ops.convnext_mlp(t.view(-1, C), bp["w1f"], bp["c1"], bp["w2"], bp["b2"], bp["gamma"], x.view(-1, C), 1e-6)
            return x
        # The 4C hidden map can be larger than what stays in L2 next to everything else: pwconv1 -> pwconv2 then pays an HBM round trip
        # for it.  Running the pair per band of rows with one band-sized hidden buffer quadruples the launches on a quarter of the rows
        # each, so the whole map goes through at once.
        hid = self.buf(tag + ".h", (B, H, W, 4 * C))
        if self.ln_fold and C % 32 == 0:
            rs = self._row_stats(B * H * W)
            t = ops.dwconv7(x, bp["dw"], bp["dwb"], out=self.buf(tag + ".t", x.shape), ln_stats=rs, work_counter=self._ctr())
            self.conv(t, bp["w1f"], 1, bias=bp["c1"], act=ACT_GELU, out=hid, row_stats=rs, col_s=bp["s1"], row_eps=1e-6)
        else:
            # two launches: the depthwise kernel + a row LayerNorm on the L2-resident result (the fused one-CTA-per-pixel-tile kernel
            # ops.dwconv7_ln needs 2.3x the instructions per output)
            t = ops.dwconv7_mma(x, bp["dwm"], out=self.buf(tag + ".t", x.shape), work_counter=self._ctr())
            ops.layernorm(t.view(-1, C), bp["lnw"], bp["lnb"], 1e-6, out=t.view(-1, C))
            self.conv(t, bp["w1"], 1, bias=bp["b1"], act=ACT_GELU, out=hid)
        self.conv(hid, bp["w2"], 1, bias=bp["b2"], gamma=bp["gamma"], res=x, out=x)
        return x

    def csp(self, x, cp, out, tag):
        """CSPLayer (network_blocks.py:147-185) on a NHWC (possibly concatenated) buffer x -> out."""
        B, H, W, _ = x.shape
        hdim = cp["c12"].cout // 2
        cat = self.buf(tag + ".cat", (B, H, W, 2 * hdim))
        self.conv_gn(x, cp["c12"], cat)  # [x_1 | x_2]
        cur = cat[..., :hdim]
        for i, (c1, c2) in enumerate(cp["m"]):
            t = self.conv_gn(cur, c1, self.buf(tag + ".m1", (B, H, W, hdim)))
            dst = cat[..., :hdim] if i == len(cp["m"]) - 1 else self.buf(tag + f".m2_{i % 2}", (B, H, W, hdim))
            cur = self.conv_gn(t, c2, dst)
        return self.conv_gn(cat, cp["c3"], out)

    # ------------------------------------------------------------------------------------------ backbone + neck
    def backbone(self, img, tag="cur", side=None):
        """features + neck.  `side(seq_dict)` (optional) is run on a second stream concurrently with the neck: in the SOT
        frame the interaction -> upsample -> correlation chain only needs the stride-16 backbone feature."""
        feats, seq = self.features(img, tag)
        if side is None:
            return self.neck(feats, tag), seq
        main = torch.cuda.current_stream()
        if self._fork_stream is None:
            self._fork_stream = torch.cuda.Stream(device=self.dev)
        self._fork_stream.wait_stream(main)
        with torch.cuda.stream(self._fork_stream):
            side_out = side(seq)
        fpn = self.neck(feats, tag)
        main.wait_stream(self._fork_stream)
        return fpn, seq, side_out

    def features(self, img, tag="cur"):
        """img fp32 NCHW [B,3,H,W] (or uint8 HWC BGR [B,H,W,3]) -> (backbone outputs (s8, s16, s32) NHWC bf16, seq_dict{feat NHWC view, h, w}).
        The s8 / s16 outputs are written straight into their slots of the neck's concat buffers (yolo_pafpn_new.py:137-155)."""
        inc = self.inc
        if img.dtype == torch.uint8:  # HWC BGR frame straight from the decoder / cv2.resize
            B, H, W, _ = img.shape
        else:
            B, _, H, W = img.shape
        assert B >= 1 and H % 32 == 0 and W % 32 == 0
        h8, w8, h16, w16, h32, w32 = H // 8, W // 8, H // 16, W // 16, H // 32, W // 32
        # concat buffers of the neck (producers write into slices)
        cat_p4 = self.buf(tag + ".cat_p4", (B, h16, w16, 2 * inc[1]))
        cat_p3 = self.buf(tag + ".cat_p3", (B, h8, w8, 2 * inc[0]))
        cat_n3 = self.buf(tag + ".cat_n3", (B, h16, w16, 2 * inc[0]))
        cat_n4 = self.buf(tag + ".cat_n4", (B, h32, w32, 2 * inc[1]))
        dst = (cat_p3[..., inc[0]:], cat_p4[..., inc[1]:], self.buf(tag + ".x0n", (B, h32, w32, inc[2])))
        if self.cfg["backbone"] == "resnet50":
            x = ops.resnet_stem(img, *self.P["rstem"], out=self.buf(tag + ".rstem", (B, H // 4, W // 4, 64)))
            self._resnet_layers(x, dst, tag)
        else:
            self._convnext_features(img, dst, tag)
        self._cat = dict(cat_p4=cat_p4, cat_p3=cat_p3, cat_n3=cat_n3, cat_n4=cat_n4)
        return dst, {"feat": dst[1], "h": h16, "w": w16}

    def _convnext_features(self, img, dst, tag):
        """ConvNeXt.forward_features (convnext.py:141-154): stages 1-3 through their out-norms into dst."""
        P, d = self.P, self.dims
        x = ops.stem_ln(img, *P["stem"])
        for i in range(4):
            if i > 0:
                lw, lb, cw, cb = P[f"down{i}"]
                Bx, Hx, Wx, Cx = x.shape
                t = ops.layernorm(x.view(-1, Cx), lw, lb, 1e-6, out=self.buf(f"{tag}.dn{i}", (Bx * Hx * Wx, Cx))).view(Bx, Hx, Wx, Cx)
                x = self.conv(t, cw, 2, 2, 0, bias=cb, out=self.buf(f"{tag}.x{i}", (Bx, Hx // 2, Wx // 2, d[i])))
            for j, bp in enumerate(P["stages"][i]):
                self.convnext_block(x, bp, f"{tag}.s{i}")
            if i >= 1:
                nw, nb = P[f"outnorm{i}"]
                Bx, Hx, Wx, Cx = x.shape
                ops.layernorm(x.view(-1, Cx), nw, nb, 1e-6, out=_rows(dst[i - 1]))

    def _resnet_layers(self, x, dst, tag):
        """ResNet._forward_impl after the stem (backbone/resnet.py:214-224): layer1..4; the last Bottleneck of layer2/3/4 writes into
        dst.  Within a layer the blocks update one buffer in place (the residual is read by the thread that overwrites it)."""
        P = self.P
        for i, blocks in enumerate(P["layers"]):
            for j, bp in enumerate(blocks):
                last = j == len(blocks) - 1
                x = self.bottleneck(x, bp, dst[i - 1] if last and i > 0 else None, f"{tag}.l{i}")

    def bottleneck(self, x, bp, out, tag):
        """Bottleneck.forward (backbone/resnet.py:104-124) with folded BatchNorms: relu(conv1) -> relu(conv2, stride) -> conv3, + identity
        (or the folded downsample conv), then ReLU in conv3's epilogue.  out=None: the layer's buffer (in place after block 0)."""
        B, H, W, _ = x.shape
        s = bp["stride"]
        (w1, b1), (w2, b2), (w3, b3) = bp["c1"], bp["c2"], bp["c3"]
        wd = w1.shape[0]
        Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
        t1 = self.conv(x, w1, 1, bias=b1, act=ACT_RELU, out=self.buf(tag + ".t1", (B, H, W, wd)))
        t2 = self.conv(t1, w2, 3, s, 1, bias=b2, act=ACT_RELU, out=self.buf(tag + ".t2", (B, Ho, Wo, wd)))
        if "ds" in bp:
            wds, bds = bp["ds"]
            idt = self.conv(x, wds, 1, s, 0, bias=bds, out=self.buf(tag + ".x", (B, Ho, Wo, wds.shape[0])))
        else:
            idt = x
        if out is None:
            out = idt
        return self.conv(t2, w3, 1, bias=b3, act=ACT_RELU, res=idt, act_after_res=True, out=out)

    def neck(self, feats, tag="cur"):
        """YOLOPAFPNNEW.forward (yolo_pafpn_new.py:137-155) on the backbone outputs (already sitting in their concat slots);
        d[1..3] = in_channels."""
        P, d = self.P, (None,) + tuple(self.inc)
        x2n, x1n, x0n = feats
        cat_p4, cat_p3, cat_n3, cat_n4 = (self._cat[k] for k in ("cat_p4", "cat_p3", "cat_n3", "cat_n4"))
        h8, w8 = x2n.shape[1:3]
        h16, w16 = x1n.shape[1:3]
        h32, w32 = x0n.shape[1:3]
        # top-down
        fpn_out0 = self.conv_gn(x0n, P["lateral_conv0"], cat_n4[..., d[2]:])
        ops.copy_upsample(fpn_out0, cat_p4[..., :d[2]], 2)
        B = x0n.shape[0]
        f_out0 = self.csp(cat_p4, P["C3_p4"], self.buf(tag + ".f_out0", (B, h16, w16, d[2])), tag + ".C3_p4")
        fpn_out1 = self.conv_gn(f_out0, P["reduce_conv1"], cat_n3[..., d[1]:])
        ops.copy_upsample(fpn_out1, cat_p3[..., :d[1]], 2)
        pan_out2 = self.csp(cat_p3, P["C3_p3"], self.buf(tag + ".pan_out2", (B, h8, w8, d[1])), tag + ".C3_p3")
        # bottom-up
        self.conv_gn(pan_out2, P["bu_conv2"], cat_n3[..., :d[1]])
        pan_out1 = self.csp(cat_n3, P["C3_n3"], self.buf(tag + ".pan_out1", (B, h16, w16, d[2])), tag + ".C3_n3")
        self.conv_gn(pan_out1, P["bu_conv1"], cat_n4[..., :d[2]])
        pan_out0 = self.csp(cat_n4, P["C3_n4"], self.buf(tag + ".pan_out0", (B, h32, w32, d[3])), tag + ".C3_n4")
        self.dbg = dict(x2n=x2n, x1n=x1n, x0n=x0n, fpn_out0=fpn_out0, f_out0=f_out0, fpn_out1=fpn_out1, pan_out2=pan_out2,
                        pan_out1=pan_out1, pan_out0=pan_out0)
        return (pan_out2, pan_out1, pan_out0)

    # ------------------------------------------------------------------------------------------ interaction
    def pos_tokens(self, h, w):
        """[2, h*w, 256] bf16: learned pos-emb (position_encoding.py:25-36) resized to (h,w) + level embed
        (deformable_transformer.py:74).  Cached per resolution (identity bicubic of unicorn.py:249 dropped)."""
        key = (h, w)
        if key not in self._pos_cache:
            col, row = self.P["pos_tab"]
            sz = col.shape[0]
            tab = torch.cat([col.unsqueeze(0).repeat(sz, 1, 1), row.unsqueeze(1).repeat(1, sz, 1)], dim=-1).permute(2, 0, 1).contiguous()
            pos = ops.bilinear(tab.unsqueeze(0), h, w)  # [1,256,h,w] fp32
            toks = pos[0].permute(1, 2, 0).reshape(1, h * w, 256) + self.P["level_embed"].view(2, 1, 256)
            self._pos_cache[key] = (toks.to(BF16).contiguous(), pos)
        return self._pos_cache[key]

    def _pos_batch(self, h, w, B):
        """pos_tokens(h, w)[0] repeated for B images: [2, B*h*w, 256] bf16 (the GroupNorm epilogue adds it per pixel of every image)."""
        if B == 1:
            return self.pos_tokens(h, w)[0]
        key = (h, w, B)
        if key not in self._pos_cache:
            self._pos_cache[key] = self.pos_tokens(h, w)[0].repeat(1, B, 1).contiguous()
        return self._pos_cache[key]

    def project_tokens(self, feat, lvl, src_rows, q_rows):
        """bottleneck conv1x1+bias -> GN32 (unicorn.py:36-38,265) of feat [B,h,w,C]; writes `src_rows` [B*h*w, 256] and
        `q_rows = src + pos + level_embed[lvl]`."""
        B, h, w = feat.shape[:3]
        pos_lvl = self._pos_batch(h, w, B)
        self.conv_gn(feat, self.P["bottleneck"], src_rows.view(B, h, w, 256), act=ACT_NONE, add2=pos_lvl[lvl].view(B, h, w, 256),
                     out2=q_rows.view(B, h, w, 256))

    def project_ref(self, feat):
        """Projection of a fixed reference frame (level 0 of the encoder input), computed once and OWNED BY THE CALLER: several
        trackers may share one engine, each keeps its own reference (the reference repo keeps `out_dict_pre` per tracker,
        unicorn_sot.py:47).  Pass the result to interaction(ref_proj=...).  feat [B,h,w,C] -> (src, q) [B*h*w, 256] each."""
        self._tracking_only("project_ref")
        B, h, w = feat.shape[:3]
        src = torch.empty(B * h * w, 256, dtype=BF16, device=self.dev)
        q = torch.empty(B * h * w, 256, dtype=BF16, device=self.dev)
        self.begin_frame()
        self.project_tokens(feat, 0, src, q)
        return src, q

    def encoder(self, src, q, h, w):
        """One deformable encoder layer over the two frames as two levels (deformable_transformer.py:122-131,
        ops/modules/ms_deform_attn.py:94-115).  src, q: [2Bhw, 256] bf16, all images' reference rows, then all their current rows.
        Returns [2Bhw, 256] bf16 (new buffer)."""
        P = self.P
        S = src.shape[0]
        value = ops.linear(src, P["value_proj"][0], bias=P["value_proj"][1], out=self.buf("enc.value", (S, 256)))
        offlog = ops.linear(q, P["offlog"][0], bias=P["offlog"][1], out=self.buf("enc.offlog", (S, 192), F32))
        att = ops.msda_fused(value, offlog, [(h, w), (h, w)], 8, 4, out=self.buf("enc.att", (S, 256)))
        x = ops.linear(att, P["output_proj"][0], bias=P["output_proj"][1], res=src, out=self.buf("enc.x", (S, 256)))
        ops.layernorm(x, *P["norm1"], 1e-5, out=x)
        hid = ops.linear(x, P["linear1"][0], bias=P["linear1"][1], act=ACT_RELU, out=self.buf("enc.hid", (S, 1024)))
        y = ops.linear(hid, P["linear2"][0], bias=P["linear2"][1], res=x, out=self.buf("enc.y", (S, 256)))
        ops.layernorm(y, *P["norm2"], 1e-5, out=y)
        return y

    def interaction(self, feat0, feat1, ref_proj=None):
        """Unicorn.forward_deform_interact (unicorn.py:260-276) of B frame pairs: feat [B,h,w,C] -> (new_feat0, new_feat1) NHWC bf16
        [B,h,w,256].  ref_proj = project_ref(feat0) of fixed reference frames ([B*h*w, 256] each): its rows are copied in instead
        of being recomputed.  Token rows are [2][B][h*w] (all reference rows, then all current rows): every projection is one
        batched conv, and the deformable attention samples each image's own rows."""
        self._tracking_only("interaction")
        B, h, w = feat1.shape[:3]
        n = B * h * w
        src, q = self.buf("enc.src", (2 * n, 256)), self.buf("enc.q", (2 * n, 256))
        if ref_proj is None:
            self.project_tokens(feat0, 0, src[:n], q[:n])
        else:
            src[:n].copy_(ref_proj[0])
            q[:n].copy_(ref_proj[1])
        self.project_tokens(feat1, 1, src[n:], q[n:])
        y = self.encoder(src, q, h, w)
        return y[:n].view(B, h, w, 256), y[n:].view(B, h, w, 256)

    def upsample(self, feat, tag):
        """Unicorn.forward_upsample (unicorn.py:41-44,311-313): [B,h,w,256] -> embedding [B,2h,2w,128] fp16."""
        self._tracking_only("upsample")
        B, h, w, _ = feat.shape
        ps = ops.pixel_shuffle2(feat, out=self.buf(tag + ".ps", (B, 2 * h, 2 * w, 64)))
        t = self.conv(ps, self.P["up1"][0], 3, 1, 1, bias=self.P["up1"][1], act=ACT_RELU, out=self.buf(tag + ".u1", (B, 2 * h, 2 * w, 256)))
        return self.conv(t, self.P["up3"][0], 3, 1, 1, bias=self.P["up3"][1], out=self.buf(tag + ".emb", (B, 2 * h, 2 * w, 128), F16))

    # ------------------------------------------------------------------------------------------ correlation
    def propagate(self, embed_ref, embed_cur, values):
        """unicorn_sot.py:88-105: label propagation + prior pyramid.  B = 1: values fp32 [K, h8*w8] -> 3 fp32 maps [K,h,w].
        B > 1 (embeddings [B,h,w,C]): values [B, K, h8*w8] -> 3 maps [B,K,h,w], every sequence against its own reference."""
        self._tracking_only("propagate")
        B, hh, ww, C = embed_cur.shape
        if B == 1:
            K = values.shape[0]
            coarse = ops.corr_propagate(embed_ref.view(-1, C), embed_cur.view(-1, C), values, out=self.buf("corr.out", (K, hh * ww), F32))
            lead = (K,)
        else:
            K = values.shape[1]
            coarse = ops.corr_propagate(embed_ref.view(B, -1, C), embed_cur.view(B, -1, C), values,
                                        out=self.buf("corr.out", (B, K, hh * ww), F32))
            lead = (B, K)
        c0 = coarse.view(*lead, hh, ww)
        c1 = ops.bilinear(c0, hh // 2, ww // 2, 2.0, 2.0, out=self.buf("corr.p1", (*lead, hh // 2, ww // 2), F32))
        c2 = ops.bilinear(c0, hh // 4, ww // 4, 4.0, 4.0, out=self.buf("corr.p2", (*lead, hh // 4, ww // 4), F32))
        return (c0, c1, c2)

    # ------------------------------------------------------------------------------------------ head
    def mask_branch(self, fpn):
        """MaskBranch.forward with use_raft (condinst/mask_branch.py:77-96,158-162) of B images: -> (mask_feats fp32 [B,h8,w8,8],
        up_masks fp32 [B,h8,w8,144])."""
        if not self.cfg["mask"]:
            self._tracking_only("mask_branch")
        M = self.P["mask"]
        B, h, w, _ = fpn[0].shape
        x = self.conv_gn(fpn[0], M["refine"][0], self.buf("mask.x", (B, h, w, 128)), act=ACT_RELU)
        for i in (1, 2):
            _, hi, wi, _ = fpn[i].shape
            xp = self.conv_gn(fpn[i], M["refine"][i], self.buf(f"mask.r{i}", (B, hi, wi, 128)), act=ACT_RELU)
            ops.aligned_bilinear_add(xp, x, h // hi)
        t = x
        for i in range(4):
            t = self.conv_gn(t, M["tower"][i], self.buf(f"mask.t{i % 2}", (B, h, w, 128)), act=ACT_RELU)
        mf = self.conv(t, M["out"][0], 1, bias=M["out"][1], out=self.buf("mask.feats", (B, h, w, 8), F32))
        u = self.conv(x, M["up0"][0], 3, 1, 1, bias=M["up0"][1], act=ACT_RELU, out=self.buf("mask.u0", (B, h, w, 128)))
        um = self.conv(u, M["up2"][0], 1, bias=M["up2"][1], out=self.buf("mask.up", (B, h, w, 144), F32))
        return mf, um

    def head(self, fpn, priors, mode, with_masks=False, decode=True):
        """UnicornHead.forward eval branch (unicorn_head.py:267-336) + decode_outputs (:467-482) of B images.
        fpn: 3 NHWC bf16 maps [B,h,w,C]; priors: 3 fp32 maps with B*h*w elements each ([B,h,w], or [B,1,h,w] from propagate) or None
        (MOT: zero prior == no fusion term).  Returns fp32 [B, A, 5+ncls_mode].  with_masks=True (UnicornHeadMask, unicorn_head_mask.py:333-343) also runs the
        controller convs; their outputs are left in self.dyn_levels (3 x fp32 [B,h,w,176]) for ops.dynamic_masks.
        The per-level prediction maps (reg+obj fp32 [B,h,w,8], class logits fp32 [B,h,w,round_up(ncls, 8)]) and their sizes are left in
        self.head_maps for post_ops.det_candidates; decode=False skips the decoded tensor and returns None."""
        if self.det and (mode == "sot" or priors is not None or (with_masks and not self.cfg["mask"])):
            raise ValueError(f"UnicornEngine.head: {self.cfg_name} is a detector: mode 'mot' (or 'whole'), no priors"
                             + ("" if self.cfg["mask"] else ", no masks"))
        B = fpn[0].shape[0]
        self._with_masks = with_masks
        self.dyn_levels = [None] * 3
        sfx = "_sot" if mode == "sot" else ""
        ro_outs, cls_outs, hw = [None] * 3, [None] * 3, [None] * 3
        ncls = 1 if mode == "sot" else self.ncls
        # The three pyramid levels are independent chains of ~30 small kernels (level 2 has 1000 pixels = 8 M tiles):
        # run them on three streams (fork/join is captured into the CUDA graph) so they fill the SMs together.
        main = torch.cuda.current_stream()
        if self._side_streams is None:
            self._side_streams = [torch.cuda.Stream(device=self.dev) for _ in range(2)]
        for s_ in self._side_streams:  # fork before anything of the head is enqueued on the main stream
            s_.wait_stream(main)
        for k in (1, 2):
            with torch.cuda.stream(self._side_streams[k - 1]):
                self._head_level(k, fpn, priors, sfx, ro_outs, cls_outs, hw)
        self._head_level(0, fpn, priors, sfx, ro_outs, cls_outs, hw)
        for s_ in self._side_streams:  # join
            main.wait_stream(s_)
        self.head_maps = (ro_outs, cls_outs, hw)
        if not decode:
            return None
        A = sum(h * w for h, w in hw)
        return ops.head_decode(ro_outs, cls_outs, hw, STRIDES, ncls, out=self.buf(f"head.out{ncls}", (B, A, 5 + ncls), F32))

    def _head_level(self, k, fpn, priors, sfx, ro_outs, cls_outs, hw):
        if True:
            L = self.P["head"][k]
            B, h, w, _ = fpn[k].shape
            x = self.buf(f"head{k}.x", (B, h, w, 256))
            pr = priors[k].reshape(-1) if priors is not None else None
            self.conv_gn(fpn[k], L["stem"], x, prior=pr, beta=L["beta"] if pr is not None else None)
            feats = self._head_trunk(k, x)
            row, rob, cw, cb, _ = L["pred" + sfx]
            cls_outs[k] = ops.conv2d(feats[0], cw, 1, 1, bias=cb, out=self.buf(f"head{k}.clso", (B, h, w, cb.numel()), F32))
            ro_outs[k] = ops.conv2d(feats[1], row, 1, 1, bias=rob, out=self.buf(f"head{k}.roo", (B, h, w, 8), F32))
            hw[k] = (h, w)
            if self._with_masks:
                cw_, cb_ = L["ctrl"]
                self.dyn_levels[k] = self.conv(feats[1], cw_, 3, 1, 1, bias=cb_, out=self.buf(f"head{k}.dyn", (B, h, w, 176), F32))

    def _head_trunk(self, k, x):
        """Level k of the head after the stem, on its output x [B,h,w,256] (in place): the three ConvNeXt blocks, then the cls and reg
        towers.  Returns their outputs (cls, reg)."""
        L = self.P["head"][k]
        B, h, w, _ = x.shape
        for i in range(3):
            self.convnext_block(x, L["att"][i], f"head{k}.att")
        feats = []
        for name in ("cls", "reg"):
            cur = x
            for i, c in enumerate(L[name]):
                cur = self.conv_gn(cur, c, self.buf(f"head{k}.{name}{i % 2}", (B, h, w, 256)))
            feats.append(cur)
        return feats

    def head_shared(self, fpn, priors, mot=True, with_masks=False, src_of=None):
        """The head of one image's pyramid for several head images at once: with mot=True image 0 is the MOT image (mode "mot", no
        prior), then one SOT image (mode "sot") per prior plane.  fpn: 3 NHWC bf16 maps [1,h,w,C]; priors: the 3 fp32 maps of
        propagate ([K,h,w] planes in any leading shape, K >= 1).  The stem conv and its statistics run once at B = 1 and
        uc_groupnorm_apply_gather, with a table of zeros, writes all 1 + K (or K) stem outputs; the ConvNeXt blocks and towers run on
        all images together, the predictors of each mode on its batch slice.  Returns (MOT decoded [1, A, 5+ncls] or None, SOT
        decoded [K, A, 6]); every image equals head(fpn, its prior or None, its mode) at B = 1, bit for bit.
        with_masks=True (a *_mask config) also runs each level's controller conv on all images at once (the controllers are shared by
        both modes, unicorn_head_mask.py:334): self.dyn_levels holds 3 fp32 [1 + K (or K), h, w, 176] maps in image order, each image's
        equal to that of head(..., with_masks=True) at B = 1.
        src_of (a device int32 [K] table): the pyramids of n_seq images (fpn [n_seq,h,w,C]), and SOT image k reads image src_of[k].  The
        stem conv and its statistics run once at B = n_seq and uc_groupnorm_apply_gather writes the n_seq MOT images (with mot=True;
        image i reads image i) followed by the K SOT images; the table is read on the device, so a captured graph follows its
        contents.  Returns (MOT decoded [n_seq, A, 5+ncls] or None, SOT decoded [K, A, 6]); every image equals head(fpn[i:i+1], its
        prior or None, its mode) at B = 1 on its source image i, bit for bit."""
        self._tracking_only("head_shared")
        if with_masks and not self.cfg["mask"]:
            raise ValueError(f"UnicornEngine.head_shared: {self.cfg_name} has no mask head (with_masks needs a *_mask config)")
        n_src = fpn[0].shape[0]
        assert src_of is not None or n_src == 1, "head_shared: the pyramid of one image unless src_of maps the SOT images to theirs"
        n_mot = (n_src if src_of is not None else 1) if mot else 0
        n_sot = priors[0].numel() // (fpn[0].shape[1] * fpn[0].shape[2])
        assert n_sot >= 1 and all(p.numel() == n_sot * f.shape[1] * f.shape[2] for p, f in zip(priors, fpn))
        if src_of is None:  # every image reads image 0: zeroed when allocated, never written
            table = self.buf("shared.src0", (n_mot + n_sot,), torch.int32, zero=True)
        else:
            assert src_of.dtype == torch.int32 and src_of.numel() == n_sot
            table = self.buf("shared.src_of", (n_mot + n_sot,), torch.int32)  # MOT image i reads image i, then the SOT images' sources
            if n_mot:
                torch.arange(n_mot, out=table[:n_mot])
            table[n_mot:].copy_(src_of.view(-1))
        outs = {m: ([None] * 3, [None] * 3) for m in ("", "_sot")}  # (reg+obj, cls) maps per level of each mode
        hw = [None] * 3

        def level(k):
            L = self.P["head"][k]
            _, h, w, _ = fpn[k].shape
            c = L["stem"]
            st = self._stats(c.groups, n_src)
            t = self.conv(fpn[k], c.w, c.k, c.stride, (c.k - 1) // 2, bias=c.bias, out=self.buf(f"shared{k}.stem", (n_src, h, w, 256)),
                          gn_stats=st, gn_groups=c.groups)
            x = self.buf(f"head{k}.x", (n_mot + n_sot, h, w, 256))
            shared_ops.groupnorm_apply_gather(t, st, c.gw, c.gb, c.groups, c.eps, ACT_SILU, x, n_mot, table, prior=priors[k].reshape(-1),
                                              beta=L["beta"])
            feats = self._head_trunk(k, x)
            for sfx, i0, n in (("", 0, n_mot), ("_sot", n_mot, n_sot)):
                if n == 0:
                    continue
                row, rob, cw, cb, _ = L["pred" + sfx]
                cls, reg = feats[0][i0:i0 + n], feats[1][i0:i0 + n]
                outs[sfx][1][k] = ops.conv2d(cls, cw, 1, 1, bias=cb, out=self.buf(f"shared{k}.clso{sfx}", (n, h, w, cb.numel()), F32))
                outs[sfx][0][k] = ops.conv2d(reg, row, 1, 1, bias=rob, out=self.buf(f"shared{k}.roo{sfx}", (n, h, w, 8), F32))
            if with_masks:
                cw_, cb_ = L["ctrl"]
                self.dyn_levels[k] = self.conv(feats[1], cw_, 3, 1, 1, bias=cb_, out=self.buf(f"shared{k}.dyn", (n_mot + n_sot, h, w, 176), F32))
            hw[k] = (h, w)

        if with_masks:
            self.dyn_levels = [None] * 3
        # the three levels on three streams, as in head()
        main = torch.cuda.current_stream()
        if self._side_streams is None:
            self._side_streams = [torch.cuda.Stream(device=self.dev) for _ in range(2)]
        for s_ in self._side_streams:
            s_.wait_stream(main)
        for k in (1, 2):
            with torch.cuda.stream(self._side_streams[k - 1]):
                level(k)
        level(0)
        for s_ in self._side_streams:
            main.wait_stream(s_)
        A = sum(h * w for h, w in hw)
        out_mot = ops.head_decode(*outs[""], hw, STRIDES, self.ncls, out=self.buf("shared.out_mot", (n_mot, A, 5 + self.ncls), F32)) if mot else None
        out_sot = ops.head_decode(*outs["_sot"], hw, STRIDES, 1, out=self.buf("shared.out_sot", (n_sot, A, 6), F32))
        return out_mot, out_sot


def _cls_cols(ncls):
    """Columns of a class-logit map: the class count rounded up to the 8-row padding of the packed weights (8 for every tracking head)."""
    return (ncls + 7) // 8 * 8


def _rows(t):
    """[B,H,W,C] channel-slice view -> [B*H*W, C] strided rows view."""
    B, H, W, C = t.shape
    return t.as_strided((B * H * W, C), (t.stride(2), 1), t.storage_offset())

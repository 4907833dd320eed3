"""MOT per-frame driver on the H100 engine — the per-frame body of MOTEvaluator.evaluate_omni
(unicorn/evaluators/mot_evaluator.py:985-1057): `model(imgs, mode="whole")` -> postprocess -> score filter ->
interaction with the previous frame -> embedding upsample (current frame only) -> embedding sampling at the box
centres -> QuasiDenseEmbedTracker.match; with `assoc="byte"` the association is BYTETracker.update on the NMS output
(mot_evaluator.py:177-209, the ByteTrack arm of the evaluator) and the embedding branch is skipped.

The reference's per-box Python grid_sample loop, deepcopy of the frame dict and empty_cache() calls are gone.  The frame
is split in a device half and a host half:

  submit(frame)  enqueues every kernel of the frame (optionally as ONE CUDA-graph replay), then asynchronous copies of
                 (count, detections, sampled embeddings) into a pinned result slot, and records an event;
  collect()      waits for the oldest slot's event and runs the association on the host.

Nothing on the device depends on the association (the previous frame's s16 feature is the only carried state), so
`submit(t+1); collect(t)` overlaps the host association of frame t with the device work of frame t+1 — same results as
the sequential `step_tensor`, throughput max(device, host) instead of their sum.

With `assoc="byte"` the frames do not even share the s16 feature: `depth` > 1 keeps that many frames in flight ON THE DEVICE, each on
its own stream and engine context (UnicornEngine.fork(): same weights, own activations) like UnicornSOTTrack(depth=...); the detections
are identical to the one-stream driver's (tests/test_mot_gpu.py), collect() still returns them in frame order."""
import torch

from . import ops
from .engine import UnicornEngine
from .tracker import QuasiDenseEmbedTracker


class _Ctx:
    """One frame in flight of the ByteTrack arm: engine context, stream, input buffers, NMS workspace, pinned result slot, graph."""

    def __init__(self, eng, H, W, A, max_dets):
        dev = eng.dev
        self.eng, self.stream = eng, torch.cuda.Stream(device=dev)
        self.ws = ops.PostWorkspace(A, dev)
        self.img_in = torch.empty(1, 3, H, W, dtype=torch.float32, device=dev)
        self.img_in_u8 = torch.empty(1, H, W, 3, dtype=torch.uint8, device=dev)
        self.u8 = False
        self.slot = dict(cnt=torch.zeros(1, dtype=torch.int32).pin_memory(), dets=torch.zeros(max_dets, 7).pin_memory(),
                         ev=torch.cuda.Event(), scale=1.0, frame_id=0)
        self.graph, self.uses, self.last = None, 0, {}


class UnicornMOTTracker:
    def __init__(self, engine: UnicornEngine, input_size, conf=0.01, nms=0.7, score_thr=0.1, max_dets=1024, tracker=None,
                 assoc="qd", use_graph=False, depth=1):
        assert assoc in ("qd", "byte")
        assert depth == 1 or assoc == "byte", "only the ByteTrack arm has independent frames (the QD arm carries the previous s16 feature)"
        self.eng, self.input_size = engine, tuple(input_size)
        self.conf, self.nms, self.score_thr, self.max_dets = conf, nms, score_thr, max_dets
        self.assoc = assoc
        self.tracker = tracker if tracker is not None else (QuasiDenseEmbedTracker(device=engine.dev) if assoc == "qd" else None)
        assert self.tracker is not None, "assoc='byte' needs a BYTETracker instance"
        H, W = self.input_size
        A = (H // 8) * (W // 8) + (H // 16) * (W // 16) + (H // 32) * (W // 32)
        dev = engine.dev
        self.ws = ops.PostWorkspace(A, dev)
        self.img_in = torch.empty(1, 3, H, W, dtype=torch.float32, device=dev)
        self.img_in_u8 = torch.empty(1, H, W, 3, dtype=torch.uint8, device=dev)  # letterboxed BGR frame as cv2 / the decoder delivers it
        self._u8 = False
        self.feats = torch.zeros(max_dets, 128, dtype=torch.float32, device=dev)
        self.frame_id = 0       # frames submitted
        self.collected = 0      # frames associated
        # pre_dict of the reference loop (mot_evaluator.py:1014-1020): the s16 feature of the last frame THAT HAD DETECTIONS, kept in
        # its own buffer and updated by a device-side conditional copy (no host decision inside the frame)
        self._prev_feat = torch.zeros(1, H // 16, W // 16, engine.inc[1], dtype=torch.bfloat16, device=dev)
        self._has_prev = torch.zeros(1, dtype=torch.int32, device=dev)
        self._warned = False
        # two pinned result slots: at most one frame is in flight behind the one being associated
        self._slots = [dict(cnt=torch.zeros(1, dtype=torch.int32).pin_memory(), dets=torch.zeros(max_dets, 7).pin_memory(),
                            feats=torch.zeros(max_dets, 128).pin_memory(), ev=torch.cuda.Event(), scale=1.0, frame_id=0)
                       for _ in range(2)]
        self.use_graph = use_graph
        self._graphs = {}
        self.last = {}
        self.depth = depth
        self._ctxs = [_Ctx(engine if i == 0 else engine.fork(), H, W, A, max_dets) for i in range(depth)] if depth > 1 else None

    # ------------------------------------------------------------------------------------------ device half
    def _device_frame(self, parity):
        e = self.eng
        e.begin_frame()
        tag = "mot%d" % parity  # two buffer sets: the previous frame's s16 feature must survive
        fpn, seq = e.backbone(self.img_in_u8 if self._u8 else self.img_in, tag=tag)
        out = e.head(fpn, None, "mot")  # whole mode: zero priors (unicorn.py:133-139)
        dets, cnt = ops.postprocess_device(out[0], e.ncls, self.conf, self.nms, self.ws)
        emb = None
        if self.assoc == "qd":
            # first frame with detections: pre_dict = cur_dict (:1014-1015); afterwards pre_dict advances only on frames that
            # produced detections (the reference skips its whole tracking block when outputs[0] is None, :1005)
            ops.copy_rows_if(self._has_prev, seq["feat"], self._prev_feat, invert=True)
            _, f_cur = e.interaction(self._prev_feat, seq["feat"])
            emb = e.upsample(f_cur, "mot.emb")
            ops.sample_embed(emb, dets, self.max_dets, 8.0, count=cnt, out=self.feats)
            ops.copy_rows_if(cnt, seq["feat"], self._prev_feat)
            self._has_prev.bitwise_or_((cnt > 0).to(torch.int32))
        self.last = dict(embed=emb, head=out)

    def _ctx_frame(self, c):
        e = c.eng
        e.begin_frame()
        fpn, _ = e.backbone(c.img_in_u8 if c.u8 else c.img_in, tag="mot")
        out = e.head(fpn, None, "mot")
        ops.postprocess_device(out[0], e.ncls, self.conf, self.nms, c.ws)
        c.last = dict(embed=None, head=out)

    def _submit_ctx(self, frame, scale):
        assert self.frame_id - self.collected < self.depth, "collect() a frame first"
        c = self._ctxs[self.frame_id % self.depth]
        self.frame_id += 1
        c.stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(c.stream):
            u8 = frame.dtype == torch.uint8
            if u8 != c.u8:
                c.u8, c.graph, c.uses = u8, None, 0
            (c.img_in_u8 if u8 else c.img_in).copy_(frame, non_blocking=True)
            c.uses += 1
            if self.use_graph and c.uses > 1:  # a context's first frame runs eagerly (plan-time autotuning, buffer allocation)
                if c.graph is None:
                    torch.cuda.synchronize()
                    c.graph = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(c.graph, stream=c.stream):
                        self._ctx_frame(c)
                c.graph.replay()
            else:
                self._ctx_frame(c)
            s = c.slot
            s["cnt"].copy_(c.ws.count.view(-1)[:1], non_blocking=True)
            s["dets"].copy_(c.ws.dets[:self.max_dets], non_blocking=True)
            s["scale"], s["frame_id"] = scale, self.frame_id
            s["ev"].record()
        self.last = c.last

    def submit(self, frame, scale=1.0):
        """frame: preprocessed fp32 [1,3,H,W] or uint8 [1,H,W,3] (4x fewer H2D bytes; the float conversion happens in the stem
        kernel), host or device.  Enqueues the frame; returns immediately."""
        if self._ctxs is not None:
            return self._submit_ctx(frame, scale)
        assert self.frame_id - self.collected < 2, "collect() the previous frame first"
        self.frame_id += 1
        parity = self.frame_id & 1
        u8 = frame.dtype == torch.uint8
        if u8 != self._u8:
            self._u8, self._graphs = u8, {}  # the captured graphs read one of the two static input buffers
        (self.img_in_u8 if u8 else self.img_in).copy_(frame, non_blocking=True)
        if self.use_graph and self.frame_id > 2:
            g = self._graphs.get(parity)
            if g is None:  # frames 1-2 ran eagerly (plan-time autotuning, first-frame special case); 3 and 4 are captured
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                keep = self.last
                with torch.cuda.graph(g):
                    self._device_frame(parity)
                self._graphs[parity] = (g, self.last)
                self.last = keep
                g = self._graphs[parity]
            g[0].replay()
            self.last = g[1]
        else:
            self._device_frame(parity)
        s = self._slots[parity]
        n = self.max_dets
        s["cnt"].copy_(self.ws.count.view(-1)[:1], non_blocking=True)
        s["dets"].copy_(self.ws.dets[:n], non_blocking=True)
        if self.assoc == "qd":
            s["feats"].copy_(self.feats, non_blocking=True)
        s["scale"], s["frame_id"] = scale, self.frame_id
        s["ev"].record()

    # ------------------------------------------------------------------------------------------ host half
    def collect(self, img_info=None):
        """Association of the oldest submitted frame.  QDTrack: (bboxes [n,5] in original-image coordinates, ids [n]);
        ByteTrack: the list of active STracks (img_info = (height, width) of the original image)."""
        assert self.collected < self.frame_id, "nothing submitted"
        self.collected += 1
        s = self._slots[self.collected & 1] if self._ctxs is None else self._ctxs[(self.collected - 1) % self.depth].slot
        s["ev"].synchronize()
        total = int(s["cnt"][0])
        if total > self.max_dets and not self._warned:
            import warnings
            warnings.warn(f"UnicornMOTTracker: {total} detections after NMS, only the {self.max_dets} best are associated "
                          "(raise max_dets; the reference has no cap)")
            self._warned = True
        n = min(total, self.max_dets)
        d = s["dets"][:n].clone()
        if self.assoc == "byte":
            H, W = self.input_size
            info = img_info if img_info is not None else (H / s["scale"], W / s["scale"])
            return self.tracker.update(d.numpy(), info, (H, W))
        f = s["feats"][:n].clone()
        scores = d[:, 4] * d[:, 5]
        keep = scores > self.score_thr  # :1008-1012
        boxes = torch.cat([d[keep, :4] / s["scale"], scores[keep, None]], 1)
        labels = torch.ones(boxes.size(0))  # :1013 (all labels = 1)
        self.last.update(dets=d, feats=f)
        if n == 0:  # outputs[0] is None: the reference skips tracking for this frame altogether (:1005)
            return torch.zeros(0, 5), torch.zeros(0, dtype=torch.long)
        # detections exist but none may pass the score filter: match() still runs (tracklets age, backdrops are replaced)
        ob, _, oid = self.tracker.match(boxes, labels, f[keep], s["frame_id"])
        valid = oid > -1  # :1047-1053
        ob, oid = ob[valid], oid[valid]
        order = oid.sort()[1]
        return ob[order], oid[order]

    def step_tensor(self, frame, scale=1.0, img_info=None):
        """Sequential protocol of the reference: one frame in, its tracks out."""
        self.submit(frame, scale)
        return self.collect(img_info)

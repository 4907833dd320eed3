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
are identical to the one-stream driver's (tests/test_tracker_gpu.py), collect() still returns them in frame order."""
import torch

from . import ops
from .engine import UnicornEngine
from .frames import FrameSlot, Ring, in_flight
from .tracker import QuasiDenseEmbedTracker


class QDEmbedding:
    """The QDTrack embedding step of a frame, on the device: interaction of the frame's s16 feature with pre_dict's, embedding
    upsample, sampling at the detections' centres into `feats`.  pre_dict (mot_evaluator.py:1014-1020, :812-818) is the s16 feature
    of the last frame THAT HAD DETECTIONS, kept in its own buffer and updated by device-side conditional copies (no host decision
    inside the frame), so a frame that runs this step must run exactly once."""

    def __init__(self, eng, H, W, max_dets, tag):
        dev = eng.dev
        self.prev_feat = torch.zeros(1, H // 16, W // 16, eng.inc[1], dtype=torch.bfloat16, device=dev)
        self.has_prev = torch.zeros(1, dtype=torch.int32, device=dev)
        self.feats = torch.zeros(max_dets, 128, dtype=torch.float32, device=dev)
        self.max_dets, self.tag = max_dets, tag

    def __call__(self, e, feat, dets, cnt):
        """feat: the frame's s16 feature, (dets, cnt): its NMS output.  Returns the embedding map."""
        # first frame with detections: pre_dict = cur_dict (:1014-1015); afterwards pre_dict advances only on frames that
        # produced detections (the reference skips its whole tracking block when outputs[0] is None, :1005)
        ops.copy_rows_if(self.has_prev, feat, self.prev_feat, invert=True)
        _, f_cur = e.interaction(self.prev_feat, feat)
        emb = e.upsample(f_cur, self.tag)
        ops.sample_embed(emb, dets, self.max_dets, 8.0, count=cnt, out=self.feats)
        ops.copy_rows_if(cnt, feat, self.prev_feat)
        self.has_prev.bitwise_or_((cnt > 0).to(torch.int32))
        return emb


class _Slot(FrameSlot):
    """One MOT frame in flight: a frame slot plus its engine buffer tag and its pinned result."""

    def __init__(self, eng, H, W, stream, tag, max_dets, feats):
        super().__init__(eng, H, W, stream)
        self.tag = tag
        self.host_count = torch.zeros(1, dtype=torch.int32).pin_memory()
        self.host_dets = torch.zeros(max_dets, 7).pin_memory()
        self.host_feats = torch.zeros(max_dets, 128).pin_memory() if feats else None
        self.scale, self.frame_id = 1.0, 0
        self.warm_u8 = None  # input dtype the slot last ran eagerly with: its next frame with it is captured


class UnicornMOTTracker:
    def __init__(self, engine: UnicornEngine, input_size, conf=0.01, nms=0.7, score_thr=0.1, max_dets=1024, tracker=None,
                 assoc="qd", use_graph=False, depth=1):
        assert assoc in ("qd", "byte")
        assert depth == 1 or assoc == "byte", "only the ByteTrack arm has independent frames (the QD arm carries the previous s16 feature)"
        self.eng, self.input_size = engine, tuple(input_size)
        self.conf, self.nms, self.score_thr, self.max_dets = conf, nms, score_thr, max_dets  # bench.py reads max_dets
        self.assoc = assoc
        self.tracker = tracker if tracker is not None else (QuasiDenseEmbedTracker(device=engine.dev) if assoc == "qd" else None)
        assert self.tracker is not None, "assoc='byte' needs a BYTETracker instance"
        H, W = self.input_size
        self._qd = QDEmbedding(engine, H, W, max_dets, "mot.emb") if assoc == "qd" else None
        self.use_graph, self.depth = use_graph, depth
        self.frame_id = 0  # frames submitted
        self._warned = False
        self.last = {}
        make = lambda eng, stream, tag="mot": _Slot(eng, H, W, stream, tag, max_dets, assoc == "qd")  # noqa: E731
        if depth == 1:
            # two slots on this engine and the current stream, so that submit(t+1) may precede collect(t); they read one input
            # buffer and share the NMS workspace, each has its own backbone buffers (tag).  Their graphs serve odd / even frames.
            slots = [make(engine, None, "mot%d" % i) for i in range(2)]
            slots[1].img_in, slots[1].img_in_u8, slots[1].ws = slots[0].img_in, slots[0].img_in_u8, slots[0].ws
        else:
            slots = in_flight(engine, depth, make)
        self._ring = Ring(slots)
        self._ctxs = slots  # bench.py reads trk._ctxs[i]

    # bench.py writes img_in_u8 and replays _graphs[p][0] (p = 0, 1: the QD arm's parity graphs); tests read ws and feats
    img_in_u8 = property(lambda self: self._ctxs[0].img_in_u8)
    _graphs = property(lambda self: [(c.graph, c.last) for c in self._ctxs if c.graph is not None])
    ws = property(lambda self: self._ctxs[0].ws)
    feats = property(lambda self: self._qd.feats)

    # ------------------------------------------------------------------------------------------ device half
    def _frame(self, c):
        e = c.eng
        e.begin_frame()
        fpn, seq = e.backbone(c.img, tag=c.tag)
        out = e.head(fpn, None, "mot")  # whole mode: zero priors (unicorn.py:133-139)
        dets, cnt = ops.postprocess_device(out[0], e.ncls, self.conf, self.nms, c.ws)
        c.last = dict(embed=self._qd(e, seq["feat"], dets, cnt) if self._qd else None, head=out)

    def submit(self, frame, scale=1.0):
        """frame: preprocessed fp32 [1,3,H,W] or uint8 [1,H,W,3] (4x fewer H2D bytes; the float conversion happens in the stem
        kernel), host or device.  Enqueues the frame; returns immediately."""
        c = self._ring.submit()
        self.frame_id = self._ring.submitted
        if c.stream is not None:
            c.stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(c.stream):  # None: the current stream
            c.stage(frame)
            if c.graph is not None:
                c.graph.replay()
            elif self.use_graph and c.warm_u8 == c.u8:
                # a slot's first frame ran eagerly (plan-time autotuning, buffer allocation, first-frame special case); the second
                # is captured without a warm-up run: a QD frame advances pre_dict, so it must not run twice
                c.graph, _ = c.capture(lambda: self._frame(c))
            else:
                self._frame(c)
                c.warm_u8 = c.u8
            c.host_count.copy_(c.ws.count, non_blocking=True)
            c.host_dets.copy_(c.ws.dets[:self.max_dets], non_blocking=True)
            if self._qd:
                c.host_feats.copy_(self._qd.feats, non_blocking=True)
            c.scale, c.frame_id = scale, self.frame_id
            c.event.record()
        self.last = c.last

    # ------------------------------------------------------------------------------------------ host half
    def collect(self, img_info=None):
        """Association of the oldest submitted frame.  QDTrack: (bboxes [n,5] in original-image coordinates, ids [n]);
        ByteTrack: the list of active STracks (img_info = (height, width) of the original image)."""
        c = self._ring.collect()
        c.event.synchronize()
        total = int(c.host_count[0])
        if total > self.max_dets and not self._warned:
            import warnings
            warnings.warn(f"UnicornMOTTracker: {total} detections after NMS, only the {self.max_dets} best are associated "
                          "(raise max_dets; the reference has no cap)")
            self._warned = True
        n = min(total, self.max_dets)
        d = c.host_dets[:n].clone()
        if self.assoc == "byte":
            H, W = self.input_size
            info = img_info if img_info is not None else (H / c.scale, W / c.scale)
            return self.tracker.update(d.numpy(), info, (H, W))
        f = c.host_feats[:n].clone()
        scores = d[:, 4] * d[:, 5]
        keep = scores > self.score_thr  # :1008-1012
        boxes = torch.cat([d[keep, :4] / c.scale, scores[keep, None]], 1)
        labels = torch.ones(boxes.size(0))  # :1013 (all labels = 1)
        self.last.update(dets=d, feats=f)
        if n == 0:  # outputs[0] is None: the reference skips tracking for this frame altogether (:1005)
            return torch.zeros(0, 5), torch.zeros(0, dtype=torch.long)
        # detections exist but none may pass the score filter: match() still runs (tracklets age, backdrops are replaced)
        ob, _, oid = self.tracker.match(boxes, labels, f[keep], c.frame_id)
        valid = oid > -1  # :1047-1053
        ob, oid = ob[valid], oid[valid]
        order = oid.sort()[1]
        return ob[order], oid[order]

    def step_tensor(self, frame, scale=1.0, img_info=None):
        """Sequential protocol of the reference: one frame in, its tracks out."""
        self.submit(frame, scale)
        return self.collect(img_info)

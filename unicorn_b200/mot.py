"""MOT per-frame driver on the H100 engine — the per-frame body of MOTEvaluator.evaluate_omni
(unicorn/evaluators/mot_evaluator.py:985-1057): `model(imgs, mode="whole")` -> postprocess -> score filter ->
interaction with the previous frame -> embedding upsample (current frame only) -> embedding sampling at the box
centres -> QuasiDenseEmbedTracker.match; with `assoc="byte"` the association is BYTETracker.update on the NMS output
(mot_evaluator.py:177-209, the ByteTrack arm of the evaluator) and the embedding branch is skipped.

The reference's per-box Python grid_sample loop, deepcopy of the frame dict and empty_cache() calls are gone.  UnicornMOTBatch runs
`n_seq` sequences in lock step (one batched frame per step, every kernel computing each image as its B = 1 launch does) and splits a
step in a device half and a host half:

  submit(frames)  enqueues every kernel of the step (optionally as ONE CUDA-graph replay), then asynchronous copies of
                  (counts, detections, sampled embeddings) into a pinned result slot, and records an event;
  collect()       waits for the oldest slot's event and runs each sequence's association on the host.

Nothing on the device depends on the association (the previous frame's s16 feature is the only carried state), so
`submit(t+1); collect(t)` overlaps the host association of step t with the device work of step t+1 — same results as
the sequential `step_tensor`, throughput max(device, host) instead of their sum.

With `assoc="byte"` the frames do not even share the s16 feature: `depth` > 1 keeps that many steps in flight ON THE DEVICE, each on
its own stream and engine context (UnicornEngine.fork(): same weights, own activations) like UnicornSOTBatch(depth=...); the detections
are identical to the one-stream driver's (tests/test_tracker_gpu.py), collect() still returns them in step order.

UnicornMOTTracker is the n_seq = 1 case under the reference's one-sequence protocol."""
import warnings

import torch

from . import _lib, ops
from .engine import UnicornEngine
from .frames import FrameSlot, Ring, anchor_count, in_flight
from .tracker import QuasiDenseEmbedTracker


def _qd_match(tracker, d, f, scale, score_thr, frame_id):
    """The host half of a QD frame: score filter and QuasiDenseEmbedTracker.match on the NMS rows d [n,7] and their embeddings f [n,128]
    -> (bboxes [n,5] in original-image coordinates, ids [n]) ordered by id."""
    scores = d[:, 4] * d[:, 5]
    keep = scores > score_thr  # :1008-1012
    boxes = torch.cat([d[keep, :4] / scale, scores[keep, None]], 1)
    labels = torch.ones(boxes.size(0))  # :1013 (all labels = 1)
    if d.shape[0] == 0:  # outputs[0] is None: the reference skips tracking for this frame altogether (:1005)
        return torch.zeros(0, 5), torch.zeros(0, dtype=torch.long)
    # detections exist but none may pass the score filter: match() still runs (tracklets age, backdrops are replaced)
    ob, _, oid = tracker.match(boxes, labels, f[keep], frame_id)
    valid = oid > -1  # :1047-1053
    ob, oid = ob[valid], oid[valid]
    order = oid.sort()[1]
    return ob[order], oid[order]


class QDEmbedding:
    """The QDTrack embedding step of a frame of B images, on the device: interaction of each image's s16 feature with its pre_dict,
    embedding upsample, sampling at the image's detection centres into `feats` [B, n_keep, 128].  pre_dict (mot_evaluator.py:1014-1020,
    :812-818) is the s16 feature of the last frame THAT HAD DETECTIONS, kept in its own buffer and updated by device-side conditional
    copies (no host decision inside the frame), so a frame that runs this step must run exactly once.  gate (int32 [B]): image b's
    pre_dict and first-frame flag change only where gate[b] != 0 (an idle sequence keeps its state).

    first_step=True is the rule of qdtrack's test_omni.py:97-98 instead: pre_dict is set by a sequence's first step whether or not it
    had detections, then advances only on steps with detections."""

    def __init__(self, eng, H, W, n_keep, tag, batch=1, first_step=False):
        dev = eng.dev
        self.prev_feat = torch.zeros(batch, H // 16, W // 16, eng.inc[1], dtype=torch.bfloat16, device=dev)
        self.has_prev = torch.zeros(batch, dtype=torch.int32, device=dev)
        self.feats = torch.zeros(batch, n_keep, 128, dtype=torch.float32, device=dev)
        self.n_keep, self.tag, self.first_step = n_keep, tag, first_step

    def __call__(self, e, feat, dets, cnt, gate=None):
        """feat: the frame's s16 features [B,h,w,C], (dets, cnt): their NMS output.  Returns the embedding maps."""
        B = feat.shape[0]
        # first frame with detections: pre_dict = cur_dict (:1014-1015); afterwards pre_dict advances only on frames that
        # produced detections (the reference skips its whole tracking block when outputs[0] is None, :1005)
        ops.copy_rows_if(self.has_prev, feat, self.prev_feat, invert=True, gate=gate)
        _, f_cur = e.interaction(self.prev_feat, feat)
        emb = e.upsample(f_cur, self.tag)
        if B == 1:  # the one-image launch on the [A, 7] NMS rows
            ops.sample_embed(emb, dets.view(-1, 7), self.n_keep, 8.0, count=cnt, out=self.feats[0])
        else:
            ops.sample_embed(emb, dets.view(B, -1, 7), self.n_keep, 8.0, count=cnt, out=self.feats)
        ops.copy_rows_if(cnt, feat, self.prev_feat, gate=gate)
        started = cnt >= 0 if self.first_step else cnt > 0  # cnt >= 0: every image (the flag stays a device-side update)
        if gate is not None:
            started &= gate != 0
        self.has_prev.bitwise_or_(started.to(torch.int32))
        return emb


class _Slot(FrameSlot):
    """One MOT step in flight: a frame slot of n_seq images, its engine buffer tag, its pinned results and the step's inputs (which
    sequences are active, their scales, frame numbers and trackers), staged per slot so that a step in flight never reads the next
    step's values."""

    def __init__(self, eng, H, W, stream, n_seq, tag, n_keep, feats):
        super().__init__(eng, H, W, stream, batch=n_seq)
        self.tag = tag
        self.host_count = torch.zeros(n_seq, dtype=torch.int32).pin_memory()
        self.host_dets = torch.zeros(n_seq, n_keep, 7).pin_memory()
        self.host_feats = torch.zeros(n_seq, n_keep, 128).pin_memory() if feats else None
        self.host_active = torch.zeros(n_seq, dtype=torch.int32).pin_memory()
        self.active = torch.zeros(n_seq, dtype=torch.int32, device=eng.dev)  # the step's active table, read by the captured QD graph
        self.mask, self.scales, self.frame_ids, self.trackers = [False] * n_seq, [1.0] * n_seq, [0] * n_seq, [None] * n_seq
        self.warm_u8 = None  # input dtype the slot last ran eagerly with: its next step with it is captured


class UnicornMOTBatch:
    """`n_seq` MOT sequences in lock step: one batched frame per step (whole-mode backbone and head, NMS, and for the QD arm the
    conditional pre_dict update, interaction with the previous features, upsample and embedding sampling, all at B = n_seq), optionally
    captured as one CUDA graph; then each sequence's own tracker on the host.  Each sequence's results equal those of the same driver
    at n_seq = 1.

    start(i, tracker=None) begins a sequence in slot i at any time (a fresh QuasiDenseEmbedTracker for the QD arm unless one is given;
    the ByteTrack arm needs a BYTETracker); it writes only slot i's state and keeps the graphs.  A slot never started, or inactive in a
    step, runs on whatever its input holds: its pre_dict, first-frame flag, tracker and frame counter are left as they were and its
    result is None, as if its own tracker had not been stepped.

    submit(frames, scales, active) enqueues a step, collect(img_infos) associates the oldest one.  depth 1: two parity slots on the
    current stream let submit(t+1) precede collect(t), so the host association of step t overlaps the device work of step t+1.
    depth > 1 (ByteTrack arm only): that many steps in flight, each on its own stream and engine context."""

    _tag = "mot"  # engine buffer tag of the driver's activations
    _first_step = False  # QDEmbedding's pre_dict rule

    def __init__(self, engine: UnicornEngine, input_size, n_seq, conf=0.01, nms=0.7, score_thr=0.1, max_dets=1024, assoc="qd",
                 use_graph=False, depth=1):
        if n_seq < 1 or depth < 1 or assoc not in ("qd", "byte"):
            raise ValueError(f"UnicornMOTBatch: n_seq >= 1, depth >= 1 and assoc 'qd' or 'byte' (got {n_seq}, {depth}, {assoc!r})")
        if depth > 1 and assoc == "qd":
            raise ValueError("UnicornMOTBatch: only the ByteTrack arm has independent frames (the QD arm carries the previous s16 feature)")
        self.eng, self.input_size, self.n_seq = engine, tuple(input_size), n_seq
        self.conf, self.nms, self.score_thr, self.max_dets = conf, nms, score_thr, max_dets  # bench.py reads max_dets
        self.assoc, self.use_graph, self.depth = assoc, use_graph, depth
        H, W = self.input_size
        self.n_keep = min(max_dets, anchor_count(H, W))  # rows a sequence can have after NMS and that are read back
        self._qd = QDEmbedding(engine, H, W, self.n_keep, self._tag + ".emb", batch=n_seq, first_step=self._first_step) if assoc == "qd" else None
        make = lambda eng, stream, tag=self._tag: _Slot(eng, H, W, stream, n_seq, tag, self.n_keep, assoc == "qd")  # noqa: E731
        if depth == 1:
            # two parity slots on this engine and the current stream: one input buffer and one NMS workspace, own backbone buffers (tag)
            # and graph each
            slots = [make(engine, None, "%s%d" % (self._tag, i)) for i in range(2)]
            slots[1].img_in, slots[1].img_in_u8, slots[1].ws = slots[0].img_in, slots[0].img_in_u8, slots[0].ws
        else:
            slots = in_flight(engine, depth, make)
        self._ring = Ring(slots)
        self._ctxs = slots  # bench.py reads trk._ctxs[i]
        self.trackers = [None] * n_seq
        self.frame_ids = [0] * n_seq  # frames each sequence has run since its start()
        self.launches_per_frame = 0
        self.last, self.last_dets, self.last_feats = {}, [None] * n_seq, [None] * n_seq
        self._warned = False

    # bench.py writes img_in_u8 and replays _graphs[p][0] (p = 0, 1: the QD arm's parity graphs)
    img_in_u8 = property(lambda self: self._ctxs[0].img_in_u8)
    _graphs = property(lambda self: [(c.graph, c.last) for c in self._ctxs if c.graph is not None])
    ws = property(lambda self: self._ctxs[0].ws)
    # the QD arm's device state: pre_dict and first-frame flag per sequence, the sampled embeddings of the latest step
    prev_feat = property(lambda self: self._qd.prev_feat)
    has_prev = property(lambda self: self._qd.has_prev)
    feats = property(lambda self: self._qd.feats)

    def start(self, i, tracker=None):
        """Begin a new sequence in slot i: its first-frame flag and frame counter are reset and `tracker` (default: a fresh
        QuasiDenseEmbedTracker, as the reference creates one at frame_id == 1) is installed.  Steps already submitted finish with the
        slot's previous tracker."""
        if not 0 <= i < self.n_seq:
            raise ValueError(f"UnicornMOTBatch.start: slot {i} outside [0, {self.n_seq})")
        if tracker is None:
            if self.assoc == "byte":
                raise ValueError("UnicornMOTBatch.start: assoc='byte' needs a BYTETracker instance")
            tracker = QuasiDenseEmbedTracker(device=self.eng.dev)
        if self._qd is not None:
            self._qd.has_prev[i].zero_()  # stream-ordered after the steps in flight
        self.trackers[i], self.frame_ids[i] = tracker, 0

    # ------------------------------------------------------------------------------------------ device half
    _with_masks = False  # the head also runs the controller convs (UnicornBDDMOTSBatch)

    def _frame(self, c):
        e = c.eng
        e.begin_frame()
        fpn, seq = e.backbone(c.img, tag=c.tag)
        out = e.head(fpn, None, "mot", with_masks=self._with_masks)  # whole mode: zero priors (unicorn.py:133-139); [n_seq, A, 5+ncls]
        dets, cnt = ops.postprocess_device(out if self.n_seq > 1 else out[0], e.ncls, self.conf, self.nms, c.ws)
        self._after_nms(c, fpn)
        # one sequence needs no gate: a step without an active sequence does not run (submit)
        embed = self._qd(e, seq["feat"], dets, cnt, gate=c.active if self.n_seq > 1 else None) if self._qd is not None else None
        c.last = dict(embed=embed, head=out)

    def _after_nms(self, c, fpn):
        """Work of the step between NMS and the embedding step, inside its graph (UnicornBDDMOTSBatch: the masks)."""

    def _check(self, frames, scales, active):
        n, (H, W) = self.n_seq, self.input_size
        ok = torch.is_tensor(frames) and ((frames.dtype == torch.uint8 and tuple(frames.shape) == (n, H, W, 3)) or
                                          (frames.dtype == torch.float32 and tuple(frames.shape) == (n, 3, H, W)))
        if not ok:
            got = (tuple(frames.shape), frames.dtype) if torch.is_tensor(frames) else type(frames)
            raise ValueError(f"{type(self).__name__}: frames must be uint8 [{n},{H},{W},3] or float32 [{n},3,{H},{W}], got {got}")
        if scales is not None and len(scales) != n:
            raise ValueError(f"{type(self).__name__}: {len(scales)} scales for {n} sequences")
        if active is not None and len(active) != n:
            raise ValueError(f"{type(self).__name__}: active has {len(active)} entries for {n} sequences")

    def submit(self, frames, scales=None, active=None):
        """frames: preprocessed fp32 [n_seq,3,H,W] or uint8 [n_seq,H,W,3] (4x fewer H2D bytes; the float conversion happens in the stem
        kernel), host or device; scales: n_seq letterbox ratios (default 1); active: n_seq flags (default: every started slot).
        Enqueues the step; returns immediately."""
        self._check(frames, scales, active)
        n = self.n_seq
        mask = [self.trackers[i] is not None and (active is None or bool(active[i])) for i in range(n)]
        c = self._ring.submit()
        if not any(mask):  # no sequence to step: nothing is launched and every result is None
            c.mask = mask
            c.event.record()
            return
        if c.stream is not None:
            c.stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(c.stream):  # None: the current stream
            u8, graph = c.u8, c.graph
            try:
                c.stage(frames)  # the last step that can fail (e.g. frames on another device): nothing has changed before it
            except BaseException:
                self._ring.submitted -= 1
                c.u8, c.graph = u8, graph
                raise
            c.mask = mask
            for i in range(n):
                self.frame_ids[i] += c.mask[i]
            c.scales = [1.0] * n if scales is None else [float(s) for s in scales]
            c.frame_ids, c.trackers = list(self.frame_ids), list(self.trackers)
            if self._qd is not None and n > 1:
                # the slot's previous step was collected, so its pinned staging buffer is free again
                c.host_active.copy_(torch.tensor(c.mask, dtype=torch.int32))
                c.active.copy_(c.host_active, non_blocking=True)
            if c.graph is not None:
                c.graph.replay()
            elif self.use_graph and c.warm_u8 == c.u8:
                # a slot's first step ran eagerly (plan-time autotuning, buffer allocation, first-frame special case); the second is
                # captured without a warm-up run: a QD step advances pre_dict, so it must not run twice
                c.graph, self.launches_per_frame = c.capture(lambda: self._frame(c))
            else:
                l0 = _lib.LAUNCHES
                self._frame(c)
                self.launches_per_frame = _lib.LAUNCHES - l0
                c.warm_u8 = c.u8
            c.host_count.copy_(c.ws.count, non_blocking=True)
            c.host_dets.copy_(c.ws.dets.view(n, -1, 7)[:, :self.n_keep], non_blocking=True)
            if self._qd is not None:
                c.host_feats.copy_(self._qd.feats, non_blocking=True)
            c.event.record()
        self.last = c.last

    # ------------------------------------------------------------------------------------------ host half
    def collect(self, img_infos=None):
        """Association of the oldest submitted step: a list of n_seq results, None for an idle slot.  QDTrack: (bboxes [n,5] in
        original-image coordinates, ids [n]); ByteTrack: the active STracks (img_infos[i] = (height, width) of slot i's original image).
        last_dets[i] / last_feats[i] then hold the NMS rows / embeddings slot i's tracker was given in this step, None for an idle slot
        (and last_feats for the ByteTrack arm)."""
        c = self._ring.collect()
        c.event.synchronize()
        H, W = self.input_size
        res = [None] * self.n_seq
        self.last_dets, self.last_feats = [None] * self.n_seq, [None] * self.n_seq
        for i in range(self.n_seq):
            if not c.mask[i]:
                continue
            total = int(c.host_count[i])
            if total > self.max_dets and not self._warned:
                warnings.warn(f"UnicornMOTBatch: {total} detections after NMS in slot {i}, only the {self.max_dets} best are associated "
                              "(raise max_dets; the reference has no cap)")
                self._warned = True
            k = min(total, self.n_keep)
            d = c.host_dets[i, :k].clone()
            self.last_dets[i] = d
            if self.assoc == "byte":
                info = img_infos[i] if img_infos is not None and img_infos[i] is not None else (H / c.scales[i], W / c.scales[i])
                res[i] = c.trackers[i].update(d.numpy(), info, (H, W))
                continue
            f = c.host_feats[i, :k].clone()
            self.last_feats[i] = f
            res[i] = _qd_match(c.trackers[i], d, f, c.scales[i], self.score_thr, c.frame_ids[i])
        return res

    def step_tensor(self, frames, scales=None, active=None, img_infos=None):
        """Sequential protocol: one step in, its n_seq results out."""
        self.submit(frames, scales, active)
        return self.collect(img_infos)


class UnicornMOTTracker:
    """One MOT sequence: UnicornMOTBatch at n_seq = 1 (same arguments) with its slot started on `tracker`, under the reference's
    one-sequence protocol.  last: the device tensors of the latest submitted frame (embed, head) and the NMS rows / embeddings the
    tracker was given at the latest collect() (dets, feats)."""

    def __init__(self, engine: UnicornEngine, input_size, conf=0.01, nms=0.7, score_thr=0.1, max_dets=1024, tracker=None,
                 assoc="qd", use_graph=False, depth=1):
        self._b = UnicornMOTBatch(engine, input_size, 1, conf, nms, score_thr, max_dets, assoc, use_graph, depth)
        self._b.start(0, tracker)
        self.tracker = self._b.trackers[0]

    max_dets = property(lambda self: self._b.max_dets)
    _ctxs = property(lambda self: self._b._ctxs)
    img_in_u8 = property(lambda self: self._b.img_in_u8)
    _graphs = property(lambda self: self._b._graphs)
    ws = property(lambda self: self._b.ws)
    feats = property(lambda self: self._b._qd.feats[0])
    frame_id = property(lambda self: self._b.frame_ids[0])  # frames submitted
    last = property(lambda self: self._b.last)

    def submit(self, frame, scale=1.0):
        """frame: preprocessed fp32 [1,3,H,W] or uint8 [1,H,W,3], host or device.  Enqueues the frame; returns immediately."""
        self._b.submit(frame, [scale])

    def collect(self, img_info=None):
        """Association of the oldest submitted frame.  QDTrack: (bboxes [n,5] in original-image coordinates, ids [n]);
        ByteTrack: the list of active STracks (img_info = (height, width) of the original image)."""
        res = self._b.collect(None if img_info is None else [img_info])[0]
        self.last.update(dets=self._b.last_dets[0], feats=self._b.last_feats[0])
        return res

    def step_tensor(self, frame, scale=1.0, img_info=None):
        """Sequential protocol of the reference: one frame in, its tracks out."""
        self.submit(frame, scale)
        return self.collect(img_info)

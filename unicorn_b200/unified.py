"""SOT targets and MOT objects, or VOS objects and MOTS instances, with one backbone pass per video frame.

Unicorn's tracking checkpoints (unicorn_track_tiny / _large / _large_mot_challenge / _r50) serve SOT and MOT with one set of weights.
Run as two drivers (UnicornSOTTrack per target, UnicornMOTTracker), every frame computes the backbone and neck once per driver;
UnicornUnifiedBatch computes them once per video frame and shares them, for n_seq videos in one step:

  1. backbone + neck of the n_seq frames at B = n_seq;
  2. on the side stream that overlaps the neck, the SOT arm of the `max_targets` target slots at B = max_targets, as
     UnicornSOTBatch._frame runs it on each slot's video frame: interaction with the slot's reference projection, the two upsamples,
     propagate;
  3. UnicornEngine.head_shared: one stem conv per video frame for its MOT image and its targets' SOT images, the rest of the head on
     all of them at once;
  4. NMS of the MOT images (whole mode, ncls classes) and of the SOT images (one class, the first max_inst rows);
  5. QD arm: QDEmbedding, the device half of UnicornMOTBatch's QDTrack step, unchanged.

Each target's (dets, count) equals that of a UnicornSOTTrack initialised on the target's reference frame and box, and each video's
MOT output equals UnicornMOTTracker's on the same frames, bit for bit.

The step protocol is the MOT driver's: submit(t + 1) may precede collect(t), so the host association of step t overlaps the device
work of step t + 1; with use_graph the first step runs eagerly and the second is captured.  The target slots are static buffers the
graph reads: adding or removing a target writes them in place and never re-captures.

UnicornUnifiedTracker is UnicornUnifiedBatch at n_seq = 1 under the one-video protocol.

UnicornUnifiedMaskBatch does the same for the *_mask checkpoints, which serve VOS and MOTS with one set of weights: VOS object slots in
place of the SOT targets, the MOTS arm in place of the MOT arm, and the mask branch computed once for both.  The object and group
slots are one pool shared by all videos, and one uc_vos_aggregate_batched launch assembles every video's label map at its own
original size.  UnicornUnifiedMaskTracker is UnicornUnifiedMaskBatch at n_seq = 1 under the one-video protocol."""
import warnings

import numpy as np
import torch

from . import _lib, ops, shared_ops
from .engine import UnicornEngine
from .frames import FrameSlot, Ring, anchor_count
from .mot import QDEmbedding, _qd_match
from .mots import MaskEncoder, _mots_match, _mots_result
from .sot import LetterboxBatch, get_label_map, nv12_size, state_xywh, xyxy_resized
from .tracker import QuasiDenseEmbedTracker
from .tracker._stream import assoc_stream
from .vos import MAX_OBJECTS_PER_SEQUENCE, ROWS_PER_GROUP_SLOT, label_values


class _Unified:
    """What the unified drivers share: the frame check (one frame per video, n_seq videos), a step ring whose submit stages the
    frames or changes nothing, and the eager / capture / replay choice of a step."""

    def _check(self, frame):
        n, (H, W) = self.n_seq, self.input_size
        ok = torch.is_tensor(frame) and ((frame.dtype == torch.uint8 and tuple(frame.shape) == (n, H, W, 3)) or
                                         (frame.dtype == torch.float32 and tuple(frame.shape) == (n, 3, H, W)))
        if not ok:
            got = (tuple(frame.shape), frame.dtype) if torch.is_tensor(frame) else type(frame)
            raise ValueError(f"{type(self).__name__}: frame must be uint8 [{n},{H},{W},3] or float32 [{n},3,{H},{W}], got {got}")

    def _next_step(self, frame, slot_of):
        """Checks `frame`, takes the ring's next step s and stages the frame into the frame slot slot_of(s).  Returns (s, slot).  A
        frame that fails leaves the ring and the slot as they were."""
        self._check(frame)
        s = self._ring.submit()
        c = slot_of(s)
        u8, graph = c.u8, c.graph
        try:
            c.stage(frame)  # the last step that can fail: nothing has changed before it
        except BaseException:
            self._ring.submitted -= 1
            c.u8, c.graph = u8, graph
            raise
        return s, c

    def _run(self, c, frame_fn):
        """Runs frame_fn() in frame slot c: replays c's graph, or captures it, or runs eagerly."""
        if c.graph is not None:
            c.graph.replay()
        elif self.use_graph and self._warm_u8 == c.u8:
            # the first step ran eagerly (plan-time autotuning, buffer allocation); this one is captured without a warm-up run: a QD
            # step advances pre_dict, so it must not run twice
            c.graph, self.launches_per_frame = c.capture(frame_fn)
        else:
            l0 = _lib.LAUNCHES
            frame_fn()
            self.launches_per_frame = _lib.LAUNCHES - l0
            self._warm_u8 = c.u8


# ---------------------------------------------------------------------------------------------------------- several videos
class _BatchStep:
    """The pinned read-back of one submitted step of UnicornUnifiedBatch and the host values it was submitted with."""

    def __init__(self, n_seq, K, max_inst, n_keep, feats):
        self.sot_dets = torch.zeros(K, max_inst, 7).pin_memory()
        self.sot_count = torch.zeros(K, dtype=torch.int32).pin_memory()
        self.count = torch.zeros(n_seq, dtype=torch.int32).pin_memory()
        self.dets = torch.zeros(n_seq, n_keep, 7).pin_memory()
        self.feats = torch.zeros(n_seq, n_keep, 128).pin_memory() if feats else None
        self.host_active = torch.zeros(n_seq, dtype=torch.int32).pin_memory()  # staging of the step's active table
        self.event = torch.cuda.Event()
        self.mask, self.tids = [False] * n_seq, []
        self.scales, self.frame_ids, self.trackers = [1.0] * n_seq, [0] * n_seq, [None] * n_seq


class UnicornUnifiedBatch(_Unified):
    """`n_seq` videos in one step, each with any number of SOT targets plus optionally one MOT arm (mot = "qd", "byte" or None), one
    backbone pass per video frame.  SOT settings (conf, nms, max_inst) default to UnicornSOTTrack's, MOT settings (mot_conf, mot_nms,
    score_thr, max_dets) to UnicornMOTTracker's.

    start(i, tracker=None) opens video slot i (a fresh QuasiDenseEmbedTracker for the QD arm unless one is given; the ByteTrack arm
    needs a BYTETracker): its MOT state is reset and the targets of the slot's previous video are removed.

    The `max_targets` target slots are one pool shared by all videos; the device table `seq_of` gives each slot's video.
    add_target(i, tid, box_xyxy): the next frame of video i submitted in a step where video i is active becomes the target's reference
    frame; the target gives results from the following step on.  remove_target(i, tid) frees its slot.  Target ids are unique within
    a video.  Both write the slot buffers, seq_of and the device `active` table in stream order and never re-capture the graph.  A
    free slot computes on stale buffers: the `active` table zeroes its detection count and its result is dropped.

    The device half of a step is one CUDA graph: backbone + neck at B = n_seq; on the side stream the SOT arm of the target slots at
    B = max_targets, each slot's stride-16 feature gathered from its video through seq_of; head_shared(..., src_of=seq_of); NMS of the
    n_seq MOT images and of the target images; the QD arm's QDEmbedding at B = n_seq, gated by the step's active videos.

    submit(frames, scales, active) / collect(img_infos) follow UnicornMOTBatch at depth 1: submit(t + 1) may precede collect(t).  A
    video idle in a step keeps its MOT state (pre_dict, first-frame flag, tracker, frame counter), its targets report nothing and a
    pending reference waits for its next active step.  Steps already submitted report the targets that were live when they were
    submitted."""

    def __init__(self, engine: UnicornEngine, input_size, n_seq, max_targets, mot="qd", conf=0.001, nms=0.65, max_inst=3,
                 mot_conf=0.01, mot_nms=0.7, score_thr=0.1, max_dets=1024, use_graph=True):
        if engine.det:
            raise ValueError(f"UnicornUnifiedBatch: {engine.cfg_name} is a detector; SOT and MOT need a tracking config")
        if mot not in ("qd", "byte", None):
            raise ValueError(f"UnicornUnifiedBatch: mot must be 'qd', 'byte' or None (got {mot!r})")
        if n_seq < 1 or max_targets < 1:
            raise ValueError(f"UnicornUnifiedBatch: n_seq and max_targets must be >= 1 (got {n_seq}, {max_targets})")
        self.eng, self.input_size, self.n_seq, self.max_targets, self.mot = engine, tuple(input_size), n_seq, max_targets, mot
        self.conf, self.nms, self.max_inst = conf, nms, max_inst
        self.mot_conf, self.mot_nms, self.score_thr, self.max_dets = mot_conf, mot_nms, score_thr, max_dets
        self.use_graph = use_graph
        H, W = self.input_size
        dev, K = engine.dev, max_targets
        A = anchor_count(H, W)
        self.n_keep = min(max_dets, A)
        self._slot = FrameSlot(engine, H, W, batch=n_seq)  # input buffers, the MOT images' NMS workspace, the graph
        self.sot_ws = ops.PostWorkspace(A, dev, K)
        self._qd = QDEmbedding(engine, H, W, self.n_keep, "unifiedb.emb", batch=n_seq) if mot == "qd" else None
        # the target slots: reference projection and label values as UnicornSOTBatch keeps them, the device active table and each
        # slot's video
        n16 = (H // 16) * (W // 16)
        self.ref_proj = (torch.zeros(K * n16, 256, dtype=torch.bfloat16, device=dev), torch.zeros(K * n16, 256, dtype=torch.bfloat16, device=dev))
        self.lbs_pre = torch.zeros(K, 1, (H // 8) * (W // 8), dtype=torch.float32, device=dev)
        self.active = torch.zeros(K, dtype=torch.int32, device=dev)
        self.seq_of = torch.zeros(K, dtype=torch.int32, device=dev)
        self.gate = torch.zeros(n_seq, dtype=torch.int32, device=dev)  # the step's active videos, read by the QD arm
        self._tid = [None] * K  # (video, target id) per slot, live or waiting for its reference frame
        self._pending = {}  # slot -> box (resized-image xyxy) of the targets whose reference is their video's next active frame
        self._ring = Ring([_BatchStep(n_seq, K, max_inst, self.n_keep, mot == "qd") for _ in range(2)])
        self._warm_u8 = None
        self._frames = LetterboxBatch(n_seq, self.input_size, engine.dev)  # the letterboxed frames of track()
        self.started = [False] * n_seq
        self.trackers = [None] * n_seq
        self.frame_ids = [0] * n_seq  # active steps per video since its start(): the QD arm's frame number
        self.states = [{} for _ in range(n_seq)]  # track(): the reference-protocol state of every target of each video
        self.launches_per_frame = 0
        self.last = {}
        self.last_dets, self.last_feats = [None] * n_seq, [None] * n_seq
        self._warned = False

    graph = property(lambda self: self._slot.graph)

    def targets(self, i):
        """The target ids of video i, live or waiting for their reference frame, in slot order."""
        return [t[1] for t in self._tid if t is not None and t[0] == i]

    # ------------------------------------------------------------------------------------------ videos and targets
    def _check_video(self, i, what):
        if not (isinstance(i, (int, np.integer)) and 0 <= i < self.n_seq):
            raise ValueError(f"UnicornUnifiedBatch.{what}: unknown video {i!r} (n_seq = {self.n_seq})")
        if what != "start" and not self.started[i]:
            raise ValueError(f"UnicornUnifiedBatch.{what}: video {i} has not been started")

    def start(self, i, tracker=None):
        """Open video slot i: its MOT state is reset, `tracker` installed and the targets of the slot's previous video removed.  Steps
        already submitted finish with the previous video's tracker and targets."""
        self._check_video(i, "start")
        if self.mot == "byte" and tracker is None:
            raise ValueError("UnicornUnifiedBatch.start: mot='byte' needs a BYTETracker instance")
        if self.mot == "qd" and tracker is None:
            tracker = QuasiDenseEmbedTracker(device=self.eng.dev)
        for tid in self.targets(i):
            self.remove_target(i, tid)
        if self._qd is not None:
            self._qd.has_prev[i].zero_()  # stream-ordered after the steps in flight
        self.started[i], self.trackers[i], self.frame_ids[i] = True, tracker if self.mot is not None else None, 0
        self.states[i] = {}

    def _check_new(self, new):
        """new: {video: [target ids]} about to be added."""
        for i, tids in new.items():
            self._check_video(i, "add_target")
            known = set(self.targets(i))
            if len(set(tids)) != len(tids) or known & set(tids):
                raise ValueError(f"UnicornUnifiedBatch: duplicate target id of video {i} in {tids} (live: {sorted(known, key=str)})")
        n_live, n_new = sum(t is not None for t in self._tid), sum(len(t) for t in new.values())
        if n_live + n_new > self.max_targets:
            raise ValueError(f"UnicornUnifiedBatch: {n_live} + {n_new} targets exceed max_targets = {self.max_targets}")

    def add_target(self, i, tid, box_xyxy):
        """Track `tid` in video i from the box [x1, y1, x2, y2] (resized-image coordinates) in video i's next active frame."""
        self._check_new({i: [tid]})
        box = torch.as_tensor(box_xyxy, dtype=torch.float32).view(-1)
        if box.numel() != 4:
            raise ValueError(f"UnicornUnifiedBatch.add_target: box_xyxy needs 4 values (got {box.numel()})")
        k = self._tid.index(None)
        self._tid[k], self._pending[k] = (i, tid), box
        self.seq_of[k].fill_(i)  # stream-ordered after the steps in flight, which read the slot's previous video

    def remove_target(self, i, tid):
        """Stop tracking `tid` of video i and free its slot (steps already submitted still report it)."""
        self._check_video(i, "remove_target")
        if (i, tid) not in self._tid:
            raise ValueError(f"UnicornUnifiedBatch.remove_target: unknown target id {tid!r} of video {i}")
        k = self._tid.index((i, tid))
        self._tid[k] = None
        if self._pending.pop(k, None) is None:
            self.active[k].fill_(0)  # stream-ordered after the steps in flight
        self.states[i].pop(tid, None)

    def _write_references(self, boxes):
        """The targets of `boxes` (slot -> box) take their video's frame of the step just enqueued as their reference frame: the
        frame's stride-16 feature is projected once per video and written into the slots (UnicornSOTBatch.initialize_tensor on that
        feature)."""
        e = self.eng
        H, W = self.input_size
        n16 = (H // 16) * (W // 16)
        for i in sorted({self._tid[k][0] for k in boxes}):
            src, q = e.project_ref(self.last["feat"][i:i + 1])
            for k, box in boxes.items():
                if self._tid[k][0] != i:
                    continue
                self.ref_proj[0][k * n16:(k + 1) * n16].copy_(src)
                self.ref_proj[1][k * n16:(k + 1) * n16].copy_(q)
                lab = get_label_map(box, H, W, e.dev)
                self.lbs_pre[k].copy_(ops.bilinear(lab, H // 8, W // 8, 8.0, 8.0).reshape(1, -1))
                self.active[k].fill_(1)

    # ------------------------------------------------------------------------------------------ device half
    def _frame(self):
        e, c, K, n = self.eng, self._slot, self.max_targets, self.n_seq
        e.begin_frame()
        values = self.lbs_pre if K > 1 else self.lbs_pre[0]

        def correlate(seq):  # the SOT arm, on the stream that overlaps the neck: each slot pairs its reference with its video's frame
            feat = seq["feat"]
            if n > 1:  # each slot's feature from its video's frame
                feat = torch.index_select(feat, 0, self.seq_of, out=e.buf("unifiedb.featK", (K,) + tuple(feat.shape[1:])))
            elif K > 1:  # one video: a broadcast copy, measurably faster than index_select through a table of zeros
                feat = e.buf("unifiedb.featK", (K,) + tuple(feat.shape[1:])).copy_(feat.expand(K, -1, -1, -1))
            f_pre, f_cur = e.interaction(None, feat, ref_proj=self.ref_proj)
            return e.propagate(e.upsample(f_pre, "embp"), e.upsample(f_cur, "embc"), values)

        fpn, seq, priors = e.backbone(c.img, tag="unifiedb", side=correlate)
        # one video: seq_of is all zeros, which is head_shared's own fixed table (no table rebuilt every step)
        head_mot, head_sot = e.head_shared(fpn, priors, mot=self.mot is not None, src_of=self.seq_of if n > 1 else None)
        _, cnt = ops.postprocess_device(head_sot, 1, self.conf, self.nms, self.sot_ws, max_keep=self.max_inst)
        cnt.mul_(self.active)
        embed = None
        if head_mot is not None:
            dets, cnt = ops.postprocess_device(head_mot if n > 1 else head_mot[0], e.ncls, self.mot_conf, self.mot_nms, c.ws)
            if self._qd is not None:
                # one video needs no gate: a step without an active video does not run (submit)
                embed = self._qd(e, seq["feat"], dets, cnt, gate=self.gate if n > 1 else None)
        self.last = dict(fpn=fpn, feat=seq["feat"], priors=priors, head_mot=head_mot, head_sot=head_sot, embed=embed)

    def submit(self, frames, scales=None, active=None):
        """frames: preprocessed fp32 [n_seq,3,H,W] or uint8 [n_seq,H,W,3], host or device; scales: n_seq letterbox ratios (default 1);
        active: n_seq flags (default: every started video).  Enqueues the step on the current stream; returns immediately."""
        n = self.n_seq
        self._check(frames)
        if scales is not None and len(scales) != n:
            raise ValueError(f"UnicornUnifiedBatch: {len(scales)} scales for {n} videos")
        if active is not None and len(active) != n:
            raise ValueError(f"UnicornUnifiedBatch: active has {len(active)} entries for {n} videos")
        if active is not None and any(bool(a) and not self.started[i] for i, a in enumerate(active)):
            raise ValueError(f"UnicornUnifiedBatch: active names a video that has not been started ({list(active)}, started {self.started})")
        mask = [self.started[i] and (active is None or bool(active[i])) for i in range(n)]
        if not any(mask):  # no video to step: nothing is launched and every result is None
            s = self._ring.submit()
            s.mask = mask
            s.event.record()
            return
        s, c = self._next_step(frames, lambda s: self._slot)
        s.mask = mask
        s.tids = [None if k in self._pending or t is None or not mask[t[0]] else t for k, t in enumerate(self._tid)]
        for i in range(n):
            self.frame_ids[i] += mask[i]
        s.scales = [1.0] * n if scales is None else [float(v) for v in scales]
        s.frame_ids, s.trackers = list(self.frame_ids), list(self.trackers)
        if self._qd is not None and n > 1:
            # this parity's previous step was collected, so its pinned staging buffer is free again
            s.host_active.copy_(torch.tensor(mask, dtype=torch.int32))
            self.gate.copy_(s.host_active, non_blocking=True)
        self._run(c, self._frame)
        s.sot_count.copy_(self.sot_ws.count, non_blocking=True)
        s.sot_dets.copy_(self.sot_ws.dets.view(self.max_targets, -1, 7)[:, :self.max_inst], non_blocking=True)
        if self.mot is not None:
            s.count.copy_(c.ws.count, non_blocking=True)
            s.dets.copy_(c.ws.dets.view(n, -1, 7)[:, :self.n_keep], non_blocking=True)
        if self._qd is not None:
            s.feats.copy_(self._qd.feats, non_blocking=True)
        s.event.record()
        ready = {k: box for k, box in self._pending.items() if mask[self._tid[k][0]]}
        if ready:
            self._write_references(ready)
            for k in ready:
                del self._pending[k]

    # ------------------------------------------------------------------------------------------ host half
    def collect(self, img_infos=None):
        """Results of the oldest submitted step: one entry per video, None for a video idle in that step, otherwise {"targets": {tid:
        (dets [<= max_inst, 7], count)}, "mot": ...}.  "mot" is what UnicornMOTTracker.collect returns (QDTrack: (bboxes [n,5] in
        original-image coordinates, ids [n]); ByteTrack: the active STracks, img_infos[i] = (height, width) of video i's original
        image), None without a MOT arm.  last_dets[i] / last_feats[i] then hold the NMS rows / embeddings video i's tracker was given
        in this step."""
        s = self._ring.collect()
        s.event.synchronize()
        H, W = self.input_size
        res = [None] * self.n_seq
        self.last_dets, self.last_feats = [None] * self.n_seq, [None] * self.n_seq
        for i in range(self.n_seq):
            if not s.mask[i]:
                continue
            targets = {}
            for k, t in enumerate(s.tids):
                if t is not None and t[0] == i:
                    cnt = int(s.sot_count[k])
                    targets[t[1]] = (s.sot_dets[k, :min(cnt, self.max_inst)].clone(), cnt)
            mot = None
            if self.mot is not None:
                total = int(s.count[i])
                if total > self.max_dets and not self._warned:
                    warnings.warn(f"UnicornUnifiedBatch: {total} detections after NMS in video {i}, only the {self.max_dets} best are "
                                  "associated (raise max_dets; the reference has no cap)")
                    self._warned = True
                d = s.dets[i, :min(total, self.n_keep)].clone()
                self.last_dets[i] = d
                if self.mot == "byte":
                    info = img_infos[i] if img_infos is not None and img_infos[i] is not None else (H / s.scales[i], W / s.scales[i])
                    mot = s.trackers[i].update(d.numpy(), info, (H, W))
                else:
                    f = s.feats[i, :d.shape[0]].clone()
                    self.last_feats[i] = f
                    mot = _qd_match(s.trackers[i], d, f, s.scales[i], self.score_thr, s.frame_ids[i])
            res[i] = {"targets": targets, "mot": mot}
        return res

    def step_tensor(self, frames, scales=None, active=None, img_infos=None):
        """Sequential protocol: one step in, its results out."""
        self.submit(frames, scales, active)
        return self.collect(img_infos)

    # ------------------------------------------------------------------------------------------ reference protocol
    def track(self, images, new_targets=None, img_infos=None):
        """images: n_seq raw frames (any original sizes), RGB uint8 [h, w, 3] or NV12 uint8 [3h/2, w] (sot.letterbox_frame; the two
        may be mixed), None for an idle video; each is letterboxed once for both arms.
        new_targets {video: {tid: [x, y, w, h]}} (original-image pixels) start on this step's frame of their video.  Returns one entry
        per video, None for an idle one, otherwise {"targets": {tid: [x, y, w, h]}, "mot": ...}: each target's state as
        UnicornSOTTrack.track keeps it (a new target's is its box; a target with no detection keeps its previous state), and the MOT
        arm's result with img_infos[i] defaulting to video i's frame (height, width)."""
        n = self.n_seq
        if len(images) != n:
            raise ValueError(f"UnicornUnifiedBatch.track: {len(images)} frames for {n} videos")
        for i, im in enumerate(images):
            if im is None:
                continue
            if nv12_size(im) is None and not (getattr(im, "ndim", 0) == 3 and im.shape[2] == 3 and im.dtype == np.uint8):
                raise ValueError(f"UnicornUnifiedBatch.track: frame {i} must be an RGB uint8 [h, w, 3] array")
            if not self.started[i]:
                raise ValueError(f"UnicornUnifiedBatch.track: video {i} has not been started")
        new_targets = {i: dict(v) for i, v in (new_targets or {}).items()}
        self._check_new({i: list(v) for i, v in new_targets.items()})
        for i, v in new_targets.items():
            if images[i] is None and v:
                raise ValueError(f"UnicornUnifiedBatch.track: new targets of video {i} need its frame")
        frames, ratios, sizes = self._frames(images)
        for i, v in new_targets.items():
            for tid, xywh in v.items():
                self.add_target(i, tid, xyxy_resized(xywh, ratios[i]))
                self.states[i][tid] = list(xywh)
        infos = [None if im is None else (img_infos[i] if img_infos is not None and img_infos[i] is not None else sizes[i])
                 for i, im in enumerate(images)]
        out = self.step_tensor(frames, [r or 1.0 for r in ratios], [im is not None for im in images], infos)
        res = [None] * n
        for i, o in enumerate(out):
            if o is None:
                continue
            for tid, (dets, cnt) in o["targets"].items():
                if cnt > 0 and tid in self.states[i]:
                    self.states[i][tid] = state_xywh(dets[0], ratios[i], self.input_size)
            res[i] = {"targets": {tid: self.states[i][tid] for tid in self.targets(i)}, "mot": o["mot"]}
        return res


# ---------------------------------------------------------------------------------------------------------- one video
class UnicornUnifiedTracker:
    """Up to `max_targets` SOT targets plus optionally one MOT arm (mot = "qd", "byte" or None) on one video, one backbone pass per frame:
    UnicornUnifiedBatch at n_seq = 1 (same settings) with its video started on `tracker` (default a fresh QuasiDenseEmbedTracker; the
    ByteTrack arm needs a BYTETracker), under the one-video protocol.

    add_target(tid, box_xyxy): the next submitted frame becomes the target's reference frame.  Right after that step, its stride-16
    feature is projected (project_ref) and the box's label map resized into the target's slot; the target gives results from the
    following frame on.  remove_target(tid) frees the slot.  Steps already submitted report the targets that were live when they
    were submitted.  frame_id counts the steps submitted, with or without a MOT arm."""

    def __init__(self, engine: UnicornEngine, input_size, max_targets, mot="qd", tracker=None, conf=0.001, nms=0.65, max_inst=3,
                 mot_conf=0.01, mot_nms=0.7, score_thr=0.1, max_dets=1024, use_graph=True):
        self._b = UnicornUnifiedBatch(engine, input_size, 1, max_targets, mot, conf, nms, max_inst, mot_conf, mot_nms, score_thr,
                                      max_dets, use_graph)
        self._b.start(0, tracker)

    graph = property(lambda self: self._b.graph)
    targets = property(lambda self: self._b.targets(0))
    max_targets = property(lambda self: self._b.max_targets)
    launches_per_frame = property(lambda self: self._b.launches_per_frame)
    last = property(lambda self: self._b.last)
    last_dets = property(lambda self: self._b.last_dets[0])
    last_feats = property(lambda self: self._b.last_feats[0])
    states = property(lambda self: self._b.states[0])
    tracker = property(lambda self: self._b.trackers[0])
    frame_id = property(lambda self: self._b.frame_ids[0])
    ref_proj = property(lambda self: self._b.ref_proj)
    lbs_pre = property(lambda self: self._b.lbs_pre)
    sot_ws = property(lambda self: self._b.sot_ws)
    _ring = property(lambda self: self._b._ring)
    _pending = property(lambda self: self._b._pending)
    _slot = property(lambda self: self._b._slot)
    _tid = property(lambda self: [None if t is None else t[1] for t in self._b._tid])  # target id per slot

    def add_target(self, tid, box_xyxy):
        """Track `tid` from the box [x1, y1, x2, y2] (resized-image coordinates) in the next submitted frame."""
        self._b.add_target(0, tid, box_xyxy)

    def remove_target(self, tid):
        """Stop tracking `tid` and free its slot (steps already submitted still report it)."""
        self._b.remove_target(0, tid)

    def submit(self, frame, scale=1.0):
        """frame: preprocessed fp32 [1,3,H,W] or uint8 [1,H,W,3], host or device; scale: its letterbox ratio.  Enqueues the step on
        the current stream; returns immediately."""
        self._b.submit(frame, [scale])

    def collect(self, img_info=None):
        """Results of the oldest submitted step: {"targets": {tid: (dets [<= max_inst, 7], count)}, "mot": ...} as
        UnicornUnifiedBatch.collect gives them for one video (img_info: (height, width) of the original image)."""
        return self._b.collect([img_info])[0]

    def step_tensor(self, frame, scale=1.0, img_info=None):
        """Sequential protocol: one step in, its results out."""
        self.submit(frame, scale)
        return self.collect(img_info)

    def track(self, image_rgb, new_targets=None, img_info=None):
        """image_rgb: a raw frame, RGB uint8 [h, w, 3] or NV12 uint8 [3h/2, w] (sot.letterbox_frame), letterboxed once for both
        arms.  new_targets {tid: [x, y, w, h]} (original-image pixels)
        start on this frame.  Returns {"targets": {tid: [x, y, w, h]}, "mot": ...} with UnicornUnifiedBatch.track's state rules."""
        return self._b.track([image_rgb], {0: new_targets or {}}, [img_info])[0]


# ---------------------------------------------------------------------------------------------------------- VOS objects + MOTS, several videos
MAX_VIDEOS = 64  # UC_VOS_MAX_VIDEOS: uc_vos_aggregate_batched assembles at most this many videos in one launch


class _MaskBatchStep(FrameSlot):
    """One step of UnicornUnifiedMaskBatch in flight: its frame slot of n_seq frames and graph, the device buffers its results live in
    until the next step of the same parity (the masks of both arms, each video's label map and soft masks), its pinned read-back and
    the host values it was submitted with."""

    def __init__(self, eng, H, W, n_seq, O, max_dets, n_keep, mots, share=None):
        super().__init__(eng, H, W, batch=n_seq)
        if share is not None:  # one set of input buffers and one MOTS NMS workspace for both parities
            self.img_in, self.img_in_u8, self.ws = share.img_in, share.img_in_u8, share.ws
        dev = eng.dev
        self.vos_masks = torch.zeros(O, 1, H, W, dtype=torch.float32, device=dev)
        self.host_rows = torch.zeros(O, 8).pin_memory()  # best detection row + count of every object slot
        self.host_tables = torch.zeros(n_seq + O, dtype=torch.int32).pin_memory()  # staging of the step's gate and active tables
        self.seg, self.soft = [None] * n_seq, [None] * n_seq
        self.mots_masks = torch.zeros(n_seq, max_dets, H, W, dtype=torch.float32, device=dev) if mots else None
        self.host_count = torch.zeros(n_seq, dtype=torch.int32).pin_memory() if mots else None
        self.host_dets = torch.zeros(n_seq, n_keep, 7).pin_memory() if mots else None
        self.host_feats = torch.zeros(n_seq, n_keep, 128).pin_memory() if mots else None
        self.mask = [False] * n_seq
        self.objs = [[] for _ in range(n_seq)]  # per video: (id, object slot) of its live objects
        self.new_ids = [[] for _ in range(n_seq)]  # per video: ids entering from its init_mask
        self.frame_ids, self.trackers, self.r, self.sizes = [0] * n_seq, [None] * n_seq, [1.0] * n_seq, [None] * n_seq


class UnicornUnifiedMaskBatch(_Unified):
    """`n_seq` videos in one step, each with up to 16 VOS objects plus optionally the MOTS arm (mots=True), one backbone, neck and
    mask-branch pass per video frame.  For the *_mask checkpoints.  VOS settings (conf, nms, max_inst, d_rate) default to
    UnicornVOSTrack's, MOTS settings (mots_conf, mots_nms, score_thr, max_dets, mask_thres, mots_d_rate, min_box_area) to
    UnicornMOTSTracker's.

    start(i, orig_size, tracker=None) opens video slot i with its original (h, w), which fixes its letterbox ratio r[i] = min(H / h,
    W / w): its MOTS first-frame flag is reset in stream order, `tracker` installed (default a fresh QuasiDenseEmbedTracker) and the
    objects of the slot's previous video removed.

    The `max_objects` object slots and `max_groups` group slots are one pool shared by all videos.  add_objects(i, {id: box_xyxy},
    init_mask=None), remove_object(i, id) and objects(i) manage the objects of each video (ids 1..255 and unique within the video, at
    most 16 objects per video, 8 objects per group slot, at most one init_mask per video per step, shaped like the video's
    orig_size); the objects of one add_objects call form one group and take video i's next active frame as their reference.  With
    init_mask (uint8 [h, w] label map) they enter that step's label map from it (UnicornVOSTrack.track_tensor with new objects);
    without, they appear from the following step on (UnicornVOSTrack.initialize_tensor).  The device tables group_seq,
    obj_seq, obj_row and image_of say which video, label row and mask-branch image every slot reads; they are written in place, in
    stream order, and never re-capture a graph.  Every entry is checked on the host before it is written.

    The device half of a step is one CUDA graph per parity slot: backbone + neck at B = n_seq with the VOS arm of the group slots on
    the side stream (each slot's stride-16 feature gathered through group_seq), the mask branch at B = n_seq, head_shared(...,
    with_masks=True, src_of=obj_seq) (the n_seq MOTS images, then one image per object slot), NMS of both arms (the object counts
    multiplied by the step's `active` table: 1 for live objects of the videos active in the step), uc_dynamic_masks_batched of both
    arms, and the MOTS arm's QDEmbedding at B = n_seq gated by the step's active videos.  One uc_vos_aggregate_batched launch then
    assembles every active video with objects at its own original size; an active video without objects gets a zeroed label map.

    submit(frames, active) / collect(): two parity slots, so submit(t + 1) may precede collect(t); the first step runs eagerly and the
    next is captured; a step with no active video launches nothing.  A free object slot computes on stale buffers, skipped by the
    dynamic masks, and its detection count is zeroed; steps already submitted report the objects they were submitted with.  A video idle in a step keeps its
    MOTS state (pre_dict, first-frame flag, tracker, frame counter), its objects report nothing and its pending references wait for
    its next active frame.  Each video's results equal those of the same driver at n_seq = 1, and each object's rows, mask, the label
    map and soft masks those of one UnicornVOSTrack, the MOTS results those of UnicornMOTSTracker, bit for bit."""

    def __init__(self, engine: UnicornEngine, input_size, n_seq, max_objects, max_groups=None, mots=True,
                 conf=0.001, nms=0.65, max_inst=1, d_rate=2,
                 mots_conf=0.01, mots_nms=0.7, score_thr=0.1, max_dets=64,
                 mask_thres=0.3, mots_d_rate=2, min_box_area=100, use_graph=True):
        if engine.det or not engine.cfg["mask"]:
            raise ValueError(f"UnicornUnifiedMaskBatch: {engine.cfg_name} has no tracking mask head; VOS and MOTS need a *_mask tracking config")
        max_groups = max_objects if max_groups is None else max_groups
        if not 1 <= n_seq <= MAX_VIDEOS:
            raise ValueError(f"UnicornUnifiedMaskBatch: n_seq must be in 1..{MAX_VIDEOS} (got {n_seq})")
        if max_objects < 1 or max_groups < 1 or max_dets < 1:
            raise ValueError(f"UnicornUnifiedMaskBatch: max_objects, max_groups and max_dets must be >= 1 (got {max_objects}, {max_groups}, "
                             f"{max_dets})")
        self.eng, self.input_size, self.n_seq = engine, tuple(input_size), n_seq
        self.max_objects, self.max_groups, self.mots = max_objects, max_groups, bool(mots)
        self.conf, self.nms, self.max_inst, self.d_rate = conf, nms, max_inst, d_rate
        self.mots_conf, self.mots_nms, self.score_thr, self.max_dets = mots_conf, mots_nms, score_thr, max_dets
        self.mask_thres, self.mots_d_rate, self.min_box_area = mask_thres, mots_d_rate, min_box_area
        self.use_graph = use_graph
        H, W = self.input_size
        dev, O, G = engine.dev, max_objects, max_groups
        self.R = min(ROWS_PER_GROUP_SLOT, max_objects)  # label rows of every group slot
        n8, n16 = (H // 8) * (W // 8), (H // 16) * (W // 16)
        self.n_keep = min(max_dets, anchor_count(H, W))
        self.vos_ws = ops.PostWorkspace(anchor_count(H, W), dev, O)
        self._qd = QDEmbedding(engine, H, W, self.n_keep, "unifiedmb.emb", batch=n_seq) if mots else None
        # the dynamic-mask scratch of both launches, from the expressions the launches check: O object rows and n_seq * max_dets MOTS rows
        up, up_m = 8 // d_rate, 8 // mots_d_rate
        self._scratch = torch.empty(max(O * (1 + up * up), n_seq * max_dets * (1 + up_m * up_m) if mots else 0) * n8, dtype=torch.float32,
                                    device=dev)
        self._enc = MaskEncoder(n_seq * max_dets, dev) if mots else None
        # the group and object slots as UnicornVOSBatch keeps them; the step's tables (gate of the videos, then active of the objects)
        self.ref_proj = tuple(torch.zeros(G * n16, 256, dtype=torch.bfloat16, device=dev) for _ in range(2))
        self.lbs = torch.zeros(G, self.R, n8, dtype=torch.float32, device=dev)
        i32 = dict(dtype=torch.int32, device=dev)
        self.group_seq = torch.zeros(G, **i32)  # video whose frame each group slot reads
        self.obj_seq = torch.zeros(O, **i32)  # video whose pyramid each object slot reads (head_shared's src_of)
        self.obj_row = torch.zeros(O, **i32)  # group slot * R + label row of each object slot
        self.image_of = torch.full((O,), -1, **i32)  # mask-branch image of each object slot, -1: free (skipped)
        self._tables = torch.zeros(n_seq + O, **i32)
        self.gate, self.active = self._tables[:n_seq], self._tables[n_seq:]
        self._mots_image_of = torch.arange(n_seq, **i32)  # MOTS image i reads mask-branch image i
        self.rows = torch.zeros(O, 8, dtype=torch.float32, device=dev)
        self._gs = [0] * G  # objects (live or pending) per group slot
        self._os = [None] * O  # (video, id, group slot, label row) per object slot
        self._order = [[] for _ in range(n_seq)]  # live objects of each video in group order (UnicornVOSTrack.obj_ids)
        self._pending = [[] for _ in range(n_seq)]  # per video: groups whose reference is its next active frame: (boxes, init_mask)
        first = _MaskBatchStep(engine, H, W, n_seq, O, max_dets, self.n_keep, self.mots)
        self._ring = Ring([first, _MaskBatchStep(engine, H, W, n_seq, O, max_dets, self.n_keep, self.mots, share=first)])
        self._warm_u8 = None
        self._frames = LetterboxBatch(n_seq, self.input_size, engine.dev)  # the letterboxed frames of track()
        self.started = [False] * n_seq
        self.orig_sizes, self.r = [None] * n_seq, [1.0] * n_seq
        self.trackers = [None] * n_seq
        self.frame_ids = [0] * n_seq  # active steps per video since its start()
        self.state_pre_dicts = [{} for _ in range(n_seq)]  # track(): the reference-protocol state of every object of each video
        self.launches_per_frame = 0
        self.last = {}
        self.last_rows = [None] * n_seq
        self.last_dets, self.last_feats = [None] * n_seq, [None] * n_seq

    graphs = property(lambda self: [s.graph for s in self._ring.slots])

    def objects(self, i):
        """The object ids of video i, live (in group order) then waiting for their reference frame."""
        return self._order[i] + [o for b, _ in self._pending[i] for o in b]

    # ------------------------------------------------------------------------------------------ videos and objects
    def _check_video(self, i, what):
        if not (isinstance(i, (int, np.integer)) and 0 <= i < self.n_seq):
            raise ValueError(f"UnicornUnifiedMaskBatch.{what}: unknown video {i!r} (n_seq = {self.n_seq})")
        if what != "start" and not self.started[i]:
            raise ValueError(f"UnicornUnifiedMaskBatch.{what}: video {i} has not been started")

    def _set(self, table, k, v, lo, hi):
        """table[k] = v in stream order, after checking lo <= v < hi on the host: no entry the graph reads is ever out of range."""
        if not lo <= v < hi:
            raise AssertionError(f"UnicornUnifiedMaskBatch: table entry {v} outside [{lo}, {hi})")
        table[k].fill_(v)

    def start(self, i, orig_size, tracker=None):
        """Open video slot i with original frames of orig_size (h, w): its MOTS state is reset, `tracker` installed and the objects of
        the slot's previous video removed.  Steps already submitted finish with the previous video's tracker and objects."""
        self._check_video(i, "start")
        try:
            size = tuple(int(v) for v in orig_size)
        except (TypeError, ValueError):
            size = ()
        if len(size) != 2 or min(size) < 1:
            raise ValueError(f"UnicornUnifiedMaskBatch.start: orig_size must be (h, w) >= 1, got {orig_size!r}")
        if self.mots and tracker is None:
            tracker = QuasiDenseEmbedTracker(device=self.eng.dev)
        for oid in self.objects(i):
            self.remove_object(i, oid)
        if self._qd is not None:
            self._qd.has_prev[i].zero_()  # stream-ordered after the steps in flight
        H, W = self.input_size
        self.started[i], self.trackers[i], self.frame_ids[i] = True, tracker if self.mots else None, 0
        self.orig_sizes[i], self.r[i] = size, min(H / size[0], W / size[1])
        self.state_pre_dicts[i] = {}

    def _check_add(self, new):
        """new: {video: (boxes {id: box}, init_mask or None)} about to be added.  Raises ValueError unless all of them fit together;
        returns them with the boxes as float tensors and the masks on the device."""
        out = {}
        n_new = g_new = 0
        for i, (boxes_xyxy, init_mask) in new.items():
            self._check_video(i, "add_objects")
            boxes = {oid: torch.as_tensor(b, dtype=torch.float32).view(-1) for oid, b in dict(boxes_xyxy).items()}
            known = self.objects(i)
            try:
                vals = [int(o) for o in boxes]
            except (TypeError, ValueError):
                vals = None
            if not boxes or vals is None or any(not 1 <= v <= 255 for v in vals):
                raise ValueError(f"UnicornUnifiedMaskBatch.add_objects: ids must be 1..255 (got {list(boxes)} for video {i})")
            if len(set(vals)) != len(vals) or set(vals) & {int(o) for o in known}:
                raise ValueError(f"UnicornUnifiedMaskBatch.add_objects: duplicate object id in {list(boxes)} (video {i} tracks {known})")
            if any(b.numel() != 4 for b in boxes.values()):
                raise ValueError("UnicornUnifiedMaskBatch.add_objects: every box needs 4 values")
            if len(known) + len(boxes) > MAX_OBJECTS_PER_SEQUENCE:
                raise ValueError(f"UnicornUnifiedMaskBatch.add_objects: {len(known) + len(boxes)} objects in video {i} (at most "
                                 f"{MAX_OBJECTS_PER_SEQUENCE} in one video)")
            if init_mask is not None:
                init_mask = torch.as_tensor(init_mask)
                if init_mask.dtype != torch.uint8 or tuple(init_mask.shape) != self.orig_sizes[i]:
                    raise ValueError(f"UnicornUnifiedMaskBatch.add_objects: init_mask must be uint8 {list(self.orig_sizes[i])}, got "
                                     f"{init_mask.dtype} {list(init_mask.shape)}")
                if any(m is not None for _, m in self._pending[i]):
                    raise ValueError(f"UnicornUnifiedMaskBatch.add_objects: the next step of video {i} already has an init_mask")
            n_new += len(boxes)
            g_new += -(-len(boxes) // ROWS_PER_GROUP_SLOT)
            out[i] = (boxes, init_mask)
        if n_new > self._os.count(None):
            raise ValueError(f"UnicornUnifiedMaskBatch.add_objects: {n_new} new objects but {self._os.count(None)} of max_objects = "
                             f"{self.max_objects} slots are free")
        if g_new > self._gs.count(0):
            raise ValueError(f"UnicornUnifiedMaskBatch.add_objects: {g_new} new group slots but {self._gs.count(0)} of max_groups = "
                             f"{self.max_groups} are free")
        return out

    def _add(self, i, boxes, init_mask):
        ids = list(boxes)
        for c0 in range(0, len(ids), ROWS_PER_GROUP_SLOT):
            g = self._gs.index(0)
            chunk = ids[c0:c0 + ROWS_PER_GROUP_SLOT]
            self._gs[g] = len(chunk)
            for row, oid in enumerate(chunk):
                self._os[self._os.index(None)] = (i, oid, g, row)
        self._pending[i].append((boxes, None if init_mask is None else init_mask.to(self.eng.dev).contiguous()))

    def add_objects(self, i, boxes_xyxy, init_mask=None):
        """Track the objects {id: [x1, y1, x2, y2]} (resized-image coordinates; ids 1..255) of video i from its next active frame on.
        init_mask: uint8 [h, w] label map of that frame in which they appear (at most one per video per step)."""
        for j, (boxes, mask) in self._check_add({i: (boxes_xyxy, init_mask)}).items():
            self._add(j, boxes, mask)

    def _slot_of(self, i, oid):
        return next(k for k, o in enumerate(self._os) if o is not None and o[0] == i and o[1] == oid)

    def remove_object(self, i, oid):
        """Stop tracking `oid` of video i and free its object slot, and its group slot with the group's last object (steps already
        submitted still report it)."""
        self._check_video(i, "remove_object")
        if oid not in self.objects(i):
            raise ValueError(f"UnicornUnifiedMaskBatch.remove_object: unknown object id {oid!r} of video {i}")
        k = self._slot_of(i, oid)
        g = self._os[k][2]
        self._os[k] = None
        self._gs[g] -= 1
        if oid in self._order[i]:
            self._order[i].remove(oid)
            self._set(self.image_of, k, -1, -1, self.n_seq)  # stream-ordered after the steps in flight
        else:
            j = next(j for j, (b, _) in enumerate(self._pending[i]) if oid in b)
            del self._pending[i][j][0][oid]
            if not self._pending[i][j][0]:
                del self._pending[i][j]
        self.state_pre_dicts[i].pop(oid, None)

    def _write_references(self, videos):
        """The pending groups of `videos` take their video's frame of the step just enqueued as their reference frame: the frame's
        stride-16 feature is projected once per video, and the projection, the boxes' label values and the slot tables are written
        into the groups' slots (UnicornVOSBatch._add_group per video)."""
        e, n, G = self.eng, self.n_seq, self.max_groups
        n16 = self.ref_proj[0].shape[0] // G
        for i in videos:
            src, q = e.project_ref(self.last["feat"][i:i + 1])
            for boxes, _ in self._pending[i]:
                ids = list(boxes)
                lbs = label_values([boxes[o] for o in ids], self.input_size, e.dev)
                written = set()
                for j, oid in enumerate(ids):
                    k = self._slot_of(i, oid)
                    _, _, g, row = self._os[k]
                    if g not in written:  # row 0 of a group slot may have been removed before the reference frame
                        written.add(g)
                        self.ref_proj[0][g * n16:(g + 1) * n16].copy_(src)
                        self.ref_proj[1][g * n16:(g + 1) * n16].copy_(q)
                        self.lbs[g].zero_()
                        self._set(self.group_seq, g, i, 0, n)
                    self.lbs[g, row].copy_(lbs[j])
                    self._set(self.obj_row, k, g * self.R + row, 0, G * self.R)
                    self._set(self.obj_seq, k, i, 0, n)
                    self._set(self.image_of, k, i, 0, n)
                self._order[i] += ids
            self._pending[i] = []

    # ------------------------------------------------------------------------------------------ device half
    def _frame(self, s):
        e, n = self.eng, self.n_seq
        H, W = self.input_size
        hh, ww = H // 8, W // 8
        G, O, R = self.max_groups, self.max_objects, self.R
        F32 = torch.float32
        e.begin_frame()

        def correlate(seq):  # the VOS arm, on the stream that overlaps the neck (UnicornVOSBatch._frame)
            feat = seq["feat"]
            feat = torch.index_select(feat, 0, self.group_seq, out=e.buf("unifiedmb.featG", (G,) + tuple(feat.shape[1:]), feat.dtype))
            f_pre, f_cur = e.interaction(None, feat, ref_proj=self.ref_proj)
            e_pre, e_cur = e.upsample(f_pre, "embp"), e.upsample(f_cur, "embc")
            coarse = ops.corr_propagate(e_pre.view(G, -1, 128), e_cur.view(G, -1, 128), self.lbs, out=e.buf("unifiedmb.coarse", (G, R, hh * ww), F32))
            c0 = torch.index_select(coarse.view(G * R, hh * ww), 0, self.obj_row, out=e.buf("unifiedmb.c0", (O, hh * ww), F32)).view(O, hh, ww)
            return (c0, ops.bilinear(c0, hh // 2, ww // 2, 2.0, 2.0, out=e.buf("unifiedmb.p1", (O, hh // 2, ww // 2), F32)),
                    ops.bilinear(c0, hh // 4, ww // 4, 4.0, 4.0, out=e.buf("unifiedmb.p2", (O, hh // 4, ww // 4), F32)))

        fpn, seq, priors = e.backbone(s.img, tag="unifiedmb", side=correlate)
        mf, um = e.mask_branch(fpn)  # once per video frame: every head image reads its video's
        head_mots, head_vos = e.head_shared(fpn, priors, mot=self.mots, with_masks=True, src_of=self.obj_seq)
        n_mot = n if self.mots else 0
        dyn = list(e.dyn_levels)
        hw = [(t.shape[1], t.shape[2]) for t in dyn]
        _, cnt = ops.postprocess_device(head_vos, 1, self.conf, self.nms, self.vos_ws, max_keep=self.max_inst)
        cnt.mul_(self.active)
        s.vos_masks.zero_()  # an object without a detection contributes an all-zero mask (unicorn_vos.py:154-155)
        up = 8 // self.d_rate
        ops.dynamic_masks(mf, um, [t[n_mot:] for t in dyn], hw, self.vos_ws, 1, up_rate=up, d_rate=self.d_rate, out=s.vos_masks,
                          scratch=self._scratch, image_of=self.image_of)
        self.rows[:, :7].copy_(self.vos_ws.dets.view(O, -1, 7)[:, 0])
        self.rows[:, 7].copy_(self.vos_ws.count)
        if self.mots:
            one = n == 1  # one video: the one-image launches; no gate (an idle step does not run)
            dets, cnt = ops.postprocess_device(head_mots[0] if one else head_mots, e.ncls, self.mots_conf, self.mots_nms, s.ws)
            ops.dynamic_masks(mf, um, [t[:n] for t in dyn], hw, s.ws, self.max_dets, up_rate=8 // self.mots_d_rate, d_rate=self.mots_d_rate,
                              out=s.mots_masks[0] if one else s.mots_masks, scratch=self._scratch, image_of=None if one else self._mots_image_of)
            self._qd(e, seq["feat"], dets, cnt, gate=None if one else self.gate)
        self.last = dict(feat=seq["feat"], mask_feats=mf, up_masks=um, priors=priors, head_mots=head_mots, head_vos=head_vos, dyn=dyn)

    def submit(self, frames, active=None):
        """frames: the n_seq letterboxed frames, preprocessed fp32 [n_seq,3,H,W] or uint8 [n_seq,H,W,3], host or device; active: n_seq
        flags (default: every started video).  Enqueues the step on the current stream; returns immediately."""
        n, O = self.n_seq, self.max_objects
        self._check(frames)
        if active is not None and len(active) != n:
            raise ValueError(f"UnicornUnifiedMaskBatch: active has {len(active)} entries for {n} videos")
        if active is not None and any(bool(a) and not self.started[i] for i, a in enumerate(active)):
            raise ValueError(f"UnicornUnifiedMaskBatch: active names a video that has not been started ({list(active)}, started {self.started})")
        mask = [self.started[i] and (active is None or bool(active[i])) for i in range(n)]
        if not any(mask):  # no video to step: nothing is launched and every result is None
            s = self._ring.submit()
            s.mask = mask
            s.event.record()
            return
        s, _ = self._next_step(frames, lambda s: s)
        s.mask = mask
        for i in range(n):
            self.frame_ids[i] += mask[i]
            s.objs[i] = [(oid, self._slot_of(i, oid)) for oid in self._order[i]] if mask[i] else []
            new = [(list(b), m) for b, m in self._pending[i] if m is not None] if mask[i] else []
            s.new_ids[i] = new[0][0] if new else []
        inits = {i: m for i in range(n) if mask[i] for _, m in self._pending[i] if m is not None}
        s.frame_ids, s.trackers, s.r, s.sizes = list(self.frame_ids), list(self.trackers), list(self.r), list(self.orig_sizes)
        # the step's tables: its active videos, and the live objects of those videos; this parity's previous step was collected, so
        # its pinned staging buffer is free again
        live = [0] * O
        for i in range(n):
            for _, k in s.objs[i]:
                live[k] = 1
        s.host_tables.copy_(torch.tensor([int(v) for v in mask] + live, dtype=torch.int32))
        self._tables.copy_(s.host_tables, non_blocking=True)
        self._run(s, lambda: self._frame(s))
        s.host_rows.copy_(self.rows, non_blocking=True)
        if self.mots:
            s.host_count.copy_(s.ws.count, non_blocking=True)
            s.host_dets.copy_(s.ws.dets.view(n, -1, 7)[:, :self.n_keep], non_blocking=True)
            s.host_feats.copy_(self._qd.feats, non_blocking=True)
        # the result assembly of every active video at its own original size, in one launch after the graph: the object lists change
        # with additions, so they stay outside it
        H, W = self.input_size
        videos = []
        for i in range(n):
            if not mask[i]:
                continue
            ids = [oid for oid, _ in s.objs[i]] + s.new_ids[i]
            size = s.sizes[i]
            if s.seg[i] is None or tuple(s.seg[i].shape) != size:
                s.seg[i] = torch.zeros(size, dtype=torch.uint8, device=self.eng.dev)
            if s.soft[i] is None or s.soft[i].shape[0] < len(ids) or tuple(s.soft[i].shape[1:]) != size:
                s.soft[i] = torch.zeros(max(len(ids), 4), *size, dtype=torch.float32, device=self.eng.dev)
            if ids:
                videos.append(([s.vos_masks[k] for _, k in s.objs[i]], inits.get(i), ids, s.r[i], s.soft[i], s.seg[i]))
            else:
                s.seg[i].zero_()
        if videos:
            shared_ops.vos_aggregate_batched(videos, H, W)
        s.event.record()
        ready = [i for i in range(n) if mask[i] and self._pending[i]]
        if ready:
            self._write_references(ready)

    # ------------------------------------------------------------------------------------------ host half
    def collect(self):
        """Results of the oldest submitted step: one entry per video, None for a video idle in that step, otherwise {"vos":
        {"segmentation": uint8 [h, w], "soft": fp32 [n, h, w] (device), "objects": {id: (det_row [7] | None, mask fp32 [H, W] at
        network resolution | None)}, "ids": [...]}, "mots": the write_results_mots() tuple, or None without the MOTS arm}.  The device
        tensors stay valid until the step after the next one is submitted.  last_rows[i] / last_dets[i] / last_feats[i] then hold video i's object rows, and the NMS
        rows and embeddings its tracker was given in this step."""
        s = self._ring.collect()
        s.event.synchronize()
        n = self.n_seq
        res = [None] * n
        self.last_rows, self.last_dets, self.last_feats = [None] * n, [None] * n, [None] * n
        tracked, frames = {}, [None] * n
        for i in range(n):
            if not s.mask[i]:
                continue
            objects, rows = {}, {}
            for oid, k in s.objs[i]:
                row = s.host_rows[k].clone()
                rows[oid] = row
                objects[oid] = (row[:7], s.vos_masks[k, 0]) if row[7] > 0 else (None, None)
            self.last_rows[i] = rows
            ids = [oid for oid, _ in s.objs[i]] + s.new_ids[i]
            res[i] = {"vos": dict(segmentation=s.seg[i], soft=s.soft[i][:len(ids)], objects=objects, ids=ids), "mots": None}
            if self.mots:
                h0, w0 = s.sizes[i]
                m = min(int(s.host_count[i]), self.n_keep)
                d, f = s.host_dets[i, :m].clone(), s.host_feats[i, :m].clone()
                self.last_dets[i], self.last_feats[i] = d, f
                _, oid, mrows, emit = _mots_match(s.trackers[i], d, f, s.r[i], self.score_thr, s.frame_ids[i], self.min_box_area)
                tracked[i] = oid, emit
                frames[i] = (mrows.tolist(), emit, s.r[i], h0, w0)
        if tracked:
            stream = assoc_stream(self.eng.dev)
            with torch.cuda.stream(stream):  # not behind the next step's kernels on the main stream
                stream.wait_event(s.event)
                # the encoder waits for its strings, so the encode has read s.mots_masks before collect() returns
                rles = self._enc.batch(s.mots_masks, self.mask_thres, frames)
            for i, (oid, emit) in tracked.items():
                res[i]["mots"] = _mots_result(s.frame_ids[i], oid, emit, rles[i], *s.sizes[i])
        return res

    def step_tensor(self, frames, active=None):
        """Sequential protocol: one step in, its results out."""
        self.submit(frames, active)
        return self.collect()

    # ------------------------------------------------------------------------------------------ reference protocol
    def track(self, images, infos=None):
        """images: n_seq raw frames of their videos' original sizes, RGB uint8 [h, w, 3] or NV12 uint8 [3h/2, w] (sot.letterbox_frame;
        the two may be mixed), None for an idle video; each is letterboxed once for both arms.  infos: n_seq dicts as UnicornVOSTrack.track takes them (init_object_ids, init_bbox {id: [x, y, w, h]},
        optionally init_mask) for objects that start on this frame, or None.  Returns one entry per video, None for an idle one, otherwise {"segmentation": uint8 [h, w]
        numpy, "mots": write_results_mots() tuple or None}; state_pre_dicts[i] is kept as UnicornVOSTrack.track keeps it."""
        n = self.n_seq
        infos = list(infos) if infos is not None else [None] * n
        if len(images) != n or len(infos) != n:
            raise ValueError(f"UnicornUnifiedMaskBatch.track: {len(images)} frames and {len(infos)} infos for {n} videos")
        new = {}
        for i, im in enumerate(images):
            if im is None:
                if infos[i] and "init_object_ids" in infos[i]:
                    raise ValueError(f"UnicornUnifiedMaskBatch.track: new objects of video {i} need its frame")
                continue
            size = nv12_size(im)
            if size is None and not (getattr(im, "ndim", 0) == 3 and im.shape[2] == 3 and im.dtype == np.uint8):
                raise ValueError(f"UnicornUnifiedMaskBatch.track: frame {i} must be an RGB uint8 [h, w, 3] array")
            self._check_video(i, "track")
            size = size or tuple(im.shape[:2])
            if size != self.orig_sizes[i]:
                raise ValueError(f"UnicornUnifiedMaskBatch.track: frame {i} has size {size}, its video's is {self.orig_sizes[i]}")
            info = infos[i] or {}
            if "init_object_ids" in info:
                boxes = {oid: xyxy_resized(info["init_bbox"][oid], self.r[i]) for oid in info["init_object_ids"]}
                mask = info.get("init_mask")
                new[i] = (boxes, None if mask is None else torch.as_tensor(mask).to(torch.uint8))
        new = self._check_add(new)
        for i, (boxes, mask) in new.items():
            self._add(i, boxes, mask)
            for oid in infos[i]["init_object_ids"]:
                self.state_pre_dicts[i][oid] = infos[i]["init_bbox"][oid]
        frames = self._frames(images)[0]
        out = self.step_tensor(frames, [im is not None for im in images])
        res = [None] * n
        for i, o in enumerate(out):
            if o is None:
                continue
            for oid, (det, _) in o["vos"]["objects"].items():  # unicorn_vos.py:137-149 (state of the best instance, xywh ints)
                if det is not None:
                    self.state_pre_dicts[i][oid] = state_xywh(det, self.r[i], self.input_size)
            res[i] = {"segmentation": o["vos"]["segmentation"].cpu().numpy(), "mots": o["mots"]}
        return res


class UnicornUnifiedMaskTracker:
    """Up to `max_objects` VOS objects plus optionally the MOTS arm (mots=True) on one video of original size `orig_size` (h, w), one
    backbone, neck and mask-branch pass per frame: UnicornUnifiedMaskBatch at n_seq = 1 (same settings) with its video started on
    `tracker` (the MOTS arm's QuasiDenseEmbedTracker, default a fresh one), under the one-video protocol.  Both arms use the
    letterbox ratio r = min(H / h, W / w).  frame_id counts the steps submitted."""

    def __init__(self, engine: UnicornEngine, input_size, orig_size, max_objects, max_groups=None, mots=True, tracker=None,
                 conf=0.001, nms=0.65, max_inst=1, d_rate=2,
                 mots_conf=0.01, mots_nms=0.7, score_thr=0.1, max_dets=64,
                 mask_thres=0.3, mots_d_rate=2, min_box_area=100, use_graph=True):
        self._b = UnicornUnifiedMaskBatch(engine, input_size, 1, max_objects, max_groups, mots, conf, nms, max_inst, d_rate, mots_conf,
                                          mots_nms, score_thr, max_dets, mask_thres, mots_d_rate, min_box_area, use_graph)
        self._b.start(0, orig_size, tracker)

    objects = property(lambda self: self._b.objects(0))
    frame_id = property(lambda self: self._b.frame_ids[0])
    graphs = property(lambda self: self._b.graphs)
    launches_per_frame = property(lambda self: self._b.launches_per_frame)
    last = property(lambda self: self._b.last)
    last_rows = property(lambda self: self._b.last_rows[0])
    last_dets = property(lambda self: self._b.last_dets[0])
    last_feats = property(lambda self: self._b.last_feats[0])
    state_pre_dict = property(lambda self: self._b.state_pre_dicts[0])
    r = property(lambda self: self._b.r[0])
    ref_proj = property(lambda self: self._b.ref_proj)
    lbs = property(lambda self: self._b.lbs)
    obj_row = property(lambda self: self._b.obj_row)
    active = property(lambda self: self._b.active)
    vos_ws = property(lambda self: self._b.vos_ws)
    R = property(lambda self: self._b.R)
    _ring = property(lambda self: self._b._ring)

    def add_objects(self, boxes_xyxy, init_mask=None):
        """Track the objects {id: [x1, y1, x2, y2]} (resized-image coordinates; ids 1..255) from the next submitted frame on.
        init_mask: uint8 [h, w] label map of that frame in which they appear (at most one per step)."""
        self._b.add_objects(0, boxes_xyxy, init_mask)

    def remove_object(self, oid):
        """Stop tracking `oid` and free its object slot, and its group slot with the group's last object (steps already submitted
        still report it)."""
        self._b.remove_object(0, oid)

    def submit(self, frame):
        """frame: the letterboxed frame, preprocessed fp32 [1,3,H,W] or uint8 [1,H,W,3], host or device.  Enqueues the step on the
        current stream; returns immediately."""
        self._b.submit(frame)

    def collect(self):
        """Results of the oldest submitted step: {"vos": ..., "mots": ...} as UnicornUnifiedMaskBatch.collect gives them for one
        video."""
        return self._b.collect()[0]

    def step_tensor(self, frame):
        """Sequential protocol: one step in, its results out."""
        self.submit(frame)
        return self.collect()

    def track(self, image_rgb, info=None):
        """image_rgb: a raw frame of the original size, RGB uint8 [h, w, 3] or NV12 uint8 [3h/2, w] (sot.letterbox_frame), letterboxed
        once for both arms.  info: UnicornVOSTrack's dict (init_object_ids, init_bbox {id: [x, y, w, h]}, optionally init_mask) for
        objects that start on this frame.  Returns {"segmentation": uint8 [h, w] numpy, "mots": write_results_mots() tuple or None};
        state_pre_dict is kept as UnicornVOSTrack.track keeps it."""
        return self._b.track([image_rgb], [info])[0]

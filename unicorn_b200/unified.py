"""SOT targets and MOT objects of one video with one backbone pass per frame.

Unicorn's tracking checkpoints (unicorn_track_tiny / _large / _large_mot_challenge / _r50) serve SOT and MOT with one set of weights.
Run as two drivers (UnicornSOTTrack per target, UnicornMOTTracker), every frame computes the backbone and neck once per driver;
UnicornUnifiedTracker computes them once and shares them:

  1. backbone + neck of the frame at B = 1;
  2. on the side stream that overlaps the neck, the SOT arm of the `max_targets` target slots at B = max_targets, as
     UnicornSOTBatch._frame runs it: interaction with each slot's reference projection, the two upsamples, propagate;
  3. UnicornEngine.head_shared: one stem conv for the MOT image and every SOT image, the rest of the head on all of them at once;
  4. NMS of the MOT image (whole mode, ncls classes) and of the SOT images (one class, the first max_inst rows);
  5. QD arm: QDEmbedding, the device half of UnicornMOTTracker's QDTrack step, unchanged.

Each target's (dets, count) equals that of a UnicornSOTTrack initialised on the target's reference frame and box, and the MOT output
equals UnicornMOTTracker's on the same frames, bit for bit.

The step protocol is the MOT driver's: submit(t + 1) may precede collect(t), so the host association of step t overlaps the device
work of step t + 1; with use_graph the first step runs eagerly and the second is captured.  The target slots are static buffers the
graph reads: adding or removing a target writes them in place and never re-captures."""
import warnings

import torch

from . import _lib, ops
from .engine import UnicornEngine
from .frames import FrameSlot, Ring, anchor_count
from .mot import QDEmbedding, _qd_match
from .sot import get_label_map, preprocess, state_xywh, xyxy_resized
from .tracker import QuasiDenseEmbedTracker


class _Step:
    """The pinned read-back of one submitted step and the host values it was submitted with."""

    def __init__(self, K, max_inst, n_keep, feats):
        self.sot_dets = torch.zeros(K, max_inst, 7).pin_memory()
        self.sot_count = torch.zeros(K, dtype=torch.int32).pin_memory()
        self.count = torch.zeros(1, dtype=torch.int32).pin_memory()
        self.dets = torch.zeros(n_keep, 7).pin_memory()
        self.feats = torch.zeros(n_keep, 128).pin_memory() if feats else None
        self.event = torch.cuda.Event()
        self.tids, self.scale, self.frame_id, self.tracker = [], 1.0, 0, None


class UnicornUnifiedTracker:
    """Up to `max_targets` SOT targets plus optionally one MOT arm (mot = "qd", "byte" or None) on one video, one backbone pass per frame.

    SOT settings (conf, nms, max_inst) default to UnicornSOTTrack's, MOT settings (mot_conf, mot_nms, score_thr, max_dets) to
    UnicornMOTTracker's.  `tracker`: the MOT arm's host tracker (default a fresh QuasiDenseEmbedTracker; the ByteTrack arm needs a
    BYTETracker).

    add_target(tid, box_xyxy): the next submitted frame becomes the target's reference frame.  Right after that step, its stride-16
    feature is projected (project_ref) and the box's label map resized into the target's slot; the target gives results from the
    following frame on.  remove_target(tid) frees the slot.  A free slot computes on stale buffers: the device `active` table zeroes its
    detection count and its result is dropped.  Steps already submitted report the targets that were live when they were submitted."""

    def __init__(self, engine: UnicornEngine, input_size, max_targets, mot="qd", tracker=None, conf=0.001, nms=0.65, max_inst=3,
                 mot_conf=0.01, mot_nms=0.7, score_thr=0.1, max_dets=1024, use_graph=True):
        if engine.det:
            raise ValueError(f"UnicornUnifiedTracker: {engine.cfg_name} is a detector; SOT and MOT need a tracking config")
        if mot not in ("qd", "byte", None):
            raise ValueError(f"UnicornUnifiedTracker: mot must be 'qd', 'byte' or None (got {mot!r})")
        if max_targets < 1:
            raise ValueError(f"UnicornUnifiedTracker: max_targets must be >= 1 (got {max_targets})")
        if mot == "byte" and tracker is None:
            raise ValueError("UnicornUnifiedTracker: mot='byte' needs a BYTETracker instance")
        if mot == "qd" and tracker is None:
            tracker = QuasiDenseEmbedTracker(device=engine.dev)
        self.eng, self.input_size, self.max_targets, self.mot = engine, tuple(input_size), max_targets, mot
        self.tracker = tracker if mot is not None else None
        self.conf, self.nms, self.max_inst = conf, nms, max_inst
        self.mot_conf, self.mot_nms, self.score_thr, self.max_dets = mot_conf, mot_nms, score_thr, max_dets
        self.use_graph = use_graph
        H, W = self.input_size
        dev, K = engine.dev, max_targets
        A = anchor_count(H, W)
        self.n_keep = min(max_dets, A)
        self._slot = FrameSlot(engine, H, W)  # input buffers, the MOT image's NMS workspace, the graph
        self.sot_ws = ops.PostWorkspace(A, dev, K)
        self._qd = QDEmbedding(engine, H, W, self.n_keep, "unified.emb") if mot == "qd" else None
        # the target slots: reference projection and label values as UnicornSOTBatch keeps them, and the device active table
        n16 = (H // 16) * (W // 16)
        self.ref_proj = (torch.zeros(K * n16, 256, dtype=torch.bfloat16, device=dev), torch.zeros(K * n16, 256, dtype=torch.bfloat16, device=dev))
        self.lbs_pre = torch.zeros(K, 1, (H // 8) * (W // 8), dtype=torch.float32, device=dev)
        self.active = torch.zeros(K, dtype=torch.int32, device=dev)
        self._tid = [None] * K  # target id per slot, live or waiting for its reference frame
        self._pending = {}  # slot -> box (resized-image xyxy) of the targets whose reference is the next submitted frame
        # two parity steps: submit(t + 1) writes one while collect(t) reads the other
        self._ring = Ring([_Step(K, max_inst, self.n_keep, mot == "qd") for _ in range(2)])
        self._warm_u8 = None  # input dtype the last eager step ran with: the next step with it is captured
        self._host_in = torch.full((1, H, W, 3), 114, dtype=torch.uint8).pin_memory()
        self.frame_id = 0  # steps the MOT arm has run
        self.states = {}  # track(): the reference-protocol state of every target
        self.launches_per_frame = 0
        self.last = {}
        self._warned = False

    graph = property(lambda self: self._slot.graph)
    targets = property(lambda self: [t for t in self._tid if t is not None])

    # ------------------------------------------------------------------------------------------ targets
    def _check_new(self, tids):
        tids = list(tids)
        known = set(self.targets)
        if len(set(tids)) != len(tids) or known & set(tids):
            raise ValueError(f"UnicornUnifiedTracker: duplicate target id in {tids} (live: {sorted(known, key=str)})")
        if len(known) + len(tids) > self.max_targets:
            raise ValueError(f"UnicornUnifiedTracker: {len(known)} + {len(tids)} targets exceed max_targets = {self.max_targets}")

    def add_target(self, tid, box_xyxy):
        """Track `tid` from the box [x1, y1, x2, y2] (resized-image coordinates) in the next submitted frame."""
        self._check_new([tid])
        box = torch.as_tensor(box_xyxy, dtype=torch.float32).view(-1)
        if box.numel() != 4:
            raise ValueError(f"UnicornUnifiedTracker.add_target: box_xyxy needs 4 values (got {box.numel()})")
        i = self._tid.index(None)
        self._tid[i], self._pending[i] = tid, box

    def remove_target(self, tid):
        """Stop tracking `tid` and free its slot (steps already submitted still report it)."""
        if tid not in self._tid:
            raise ValueError(f"UnicornUnifiedTracker.remove_target: unknown target id {tid!r}")
        i = self._tid.index(tid)
        self._tid[i] = None
        if self._pending.pop(i, None) is None:
            self.active[i].fill_(0)  # stream-ordered after the steps in flight
        self.states.pop(tid, None)

    def _write_references(self, boxes):
        """The targets of `boxes` (slot -> box) take the step just enqueued as their reference frame (UnicornSOTBatch.initialize_tensor
        on that frame's stride-16 feature)."""
        e = self.eng
        H, W = self.input_size
        n16 = (H // 16) * (W // 16)
        src, q = e.project_ref(self.last["feat"])
        for i, box in boxes.items():
            self.ref_proj[0][i * n16:(i + 1) * n16].copy_(src)
            self.ref_proj[1][i * n16:(i + 1) * n16].copy_(q)
            lab = get_label_map(box, H, W, e.dev)
            self.lbs_pre[i].copy_(ops.bilinear(lab, H // 8, W // 8, 8.0, 8.0).reshape(1, -1))
            self.active[i].fill_(1)

    # ------------------------------------------------------------------------------------------ device half
    def _frame(self):
        e, c, K = self.eng, self._slot, self.max_targets
        e.begin_frame()
        values = self.lbs_pre if K > 1 else self.lbs_pre[0]

        def correlate(seq):  # the SOT arm, on the stream that overlaps the neck: each target slot pairs its reference with the frame
            feat = seq["feat"]
            if K > 1:
                feat = e.buf("unified.featK", (K,) + tuple(feat.shape[1:]))
                feat.copy_(seq["feat"].expand(K, -1, -1, -1))
            f_pre, f_cur = e.interaction(None, feat, ref_proj=self.ref_proj)
            return e.propagate(e.upsample(f_pre, "embp"), e.upsample(f_cur, "embc"), values)

        fpn, seq, priors = e.backbone(c.img, tag="unified", side=correlate)
        head_mot, head_sot = e.head_shared(fpn, priors, mot=self.mot is not None)
        _, cnt = ops.postprocess_device(head_sot, 1, self.conf, self.nms, self.sot_ws, max_keep=self.max_inst)
        cnt.mul_(self.active)
        embed = None
        if head_mot is not None:
            dets, cnt = ops.postprocess_device(head_mot[0], e.ncls, self.mot_conf, self.mot_nms, c.ws)
            if self._qd is not None:
                embed = self._qd(e, seq["feat"], dets, cnt)
        self.last = dict(fpn=fpn, feat=seq["feat"], priors=priors, head_mot=head_mot, head_sot=head_sot, embed=embed)

    def _check(self, frame):
        H, W = self.input_size
        ok = torch.is_tensor(frame) and ((frame.dtype == torch.uint8 and tuple(frame.shape) == (1, H, W, 3)) or
                                         (frame.dtype == torch.float32 and tuple(frame.shape) == (1, 3, H, W)))
        if not ok:
            got = (tuple(frame.shape), frame.dtype) if torch.is_tensor(frame) else type(frame)
            raise ValueError(f"UnicornUnifiedTracker: frame must be uint8 [1,{H},{W},3] or float32 [1,3,{H},{W}], got {got}")

    def submit(self, frame, scale=1.0):
        """frame: preprocessed fp32 [1,3,H,W] or uint8 [1,H,W,3], host or device; scale: its letterbox ratio.  Enqueues the step on
        the current stream; returns immediately."""
        self._check(frame)
        c = self._slot
        s = self._ring.submit()
        u8, graph = c.u8, c.graph
        try:
            c.stage(frame)  # the last step that can fail: nothing has changed before it
        except BaseException:
            self._ring.submitted -= 1
            c.u8, c.graph = u8, graph
            raise
        s.tids = [None if i in self._pending else t for i, t in enumerate(self._tid)]
        if self.mot is not None:
            self.frame_id += 1
        s.scale, s.frame_id, s.tracker = float(scale), self.frame_id, self.tracker
        if c.graph is not None:
            c.graph.replay()
        elif self.use_graph and self._warm_u8 == c.u8:
            # the first step ran eagerly (plan-time autotuning, buffer allocation); this one is captured without a warm-up run: a QD
            # step advances pre_dict, so it must not run twice
            c.graph, self.launches_per_frame = c.capture(self._frame)
        else:
            l0 = _lib.LAUNCHES
            self._frame()
            self.launches_per_frame = _lib.LAUNCHES - l0
            self._warm_u8 = c.u8
        K = self.max_targets
        s.sot_count.copy_(self.sot_ws.count, non_blocking=True)
        s.sot_dets.copy_(self.sot_ws.dets.view(K, -1, 7)[:, :self.max_inst], non_blocking=True)
        if self.mot is not None:
            s.count.copy_(c.ws.count, non_blocking=True)
            s.dets.copy_(c.ws.dets[:self.n_keep], non_blocking=True)
        if self._qd is not None:
            s.feats.copy_(self._qd.feats[0], non_blocking=True)
        s.event.record()
        if self._pending:
            self._write_references(self._pending)
            self._pending = {}

    # ------------------------------------------------------------------------------------------ host half
    def collect(self, img_info=None):
        """Results of the oldest submitted step: {"targets": {tid: (dets [<= max_inst, 7], count)}, "mot": ...}.  "mot" is what
        UnicornMOTTracker.collect returns (QDTrack: (bboxes [n,5] in original-image coordinates, ids [n]); ByteTrack: the active
        STracks, img_info = (height, width) of the original image), None without a MOT arm."""
        s = self._ring.collect()
        s.event.synchronize()
        targets = {}
        for i, tid in enumerate(s.tids):
            if tid is not None:
                n = int(s.sot_count[i])
                targets[tid] = (s.sot_dets[i, :min(n, self.max_inst)].clone(), n)
        res = None
        self.last_dets = self.last_feats = None
        if self.mot is not None:
            total = int(s.count[0])
            if total > self.max_dets and not self._warned:
                warnings.warn(f"UnicornUnifiedTracker: {total} detections after NMS, only the {self.max_dets} best are associated "
                              "(raise max_dets; the reference has no cap)")
                self._warned = True
            d = s.dets[:min(total, self.n_keep)].clone()
            self.last_dets = d
            if self.mot == "byte":
                H, W = self.input_size
                info = img_info if img_info is not None else (H / s.scale, W / s.scale)
                res = s.tracker.update(d.numpy(), info, (H, W))
            else:
                f = s.feats[:d.shape[0]].clone()
                self.last_feats = f
                res = _qd_match(s.tracker, d, f, s.scale, self.score_thr, s.frame_id)
        return {"targets": targets, "mot": res}

    def step_tensor(self, frame, scale=1.0, img_info=None):
        """Sequential protocol: one step in, its results out."""
        self.submit(frame, scale)
        return self.collect(img_info)

    # ------------------------------------------------------------------------------------------ reference protocol
    def track(self, image_rgb, new_targets=None, img_info=None):
        """image_rgb: an RGB frame (HWC uint8), letterboxed once for both arms.  new_targets {tid: [x, y, w, h]} (original-image pixels)
        start on this frame.  Returns {"targets": {tid: [x, y, w, h]}, "mot": ...}: each target's state as UnicornSOTTrack.track keeps it
        (a new target's is its box; a target with no detection keeps its previous state), and the MOT arm's result with img_info
        defaulting to the frame's (height, width)."""
        new_targets = dict(new_targets or {})
        self._check_new(new_targets)
        frame, r = preprocess(image_rgb, self.input_size, out=self._host_in)
        for tid, xywh in new_targets.items():
            self.add_target(tid, xyxy_resized(xywh, r))
            self.states[tid] = list(xywh)
        out = self.step_tensor(frame, r, img_info if img_info is not None else tuple(image_rgb.shape[:2]))
        for tid, (dets, n) in out["targets"].items():
            if n > 0 and tid in self.states:
                self.states[tid] = state_xywh(dets[0], r, self.input_size)
        return {"targets": {tid: self.states[tid] for tid in self.targets}, "mot": out["mot"]}

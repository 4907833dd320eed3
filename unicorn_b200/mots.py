"""MOTS driver on the H100 engine — the per-frame body of MOTEvaluator.evaluate_omni_mots
(unicorn/evaluators/mot_evaluator.py:776-897): whole-mode detector with the CondInst controllers -> NMS -> dynamic-conv masks of the
kept detections -> embedding sampling -> QuasiDenseEmbedTracker.match(return_index=True) -> masks of the tracked boxes in
ascending-id order, resized to the original frame, overlap free, area filter, COCO RLE.

UnicornMOTSBatch runs `n_seq` sequences in lock step under the protocol of UnicornMOTBatch (mot.py), and like the QD arm of the MOT
driver splits a step in a device half and a host half:

  submit(frames, img_sizes)  enqueues every kernel of the step (with use_graph, one CUDA-graph replay per parity slot from the
                             slot's second step on), the masks into the slot's own buffer, and asynchronous copies of (counts,
                             detections, sampled embeddings) into pinned slot memory;
  collect()                  waits for the oldest slot, runs each active sequence's association on the host, then ONE encode of
                             the tracked instances of every sequence on the device (uc_mots_encode_batched, uc_mots_encode for a
                             single frame) on the association stream, so it does not queue behind the next step; one upload of
                             order / emit and at most two host synchronises per step.

Two slots: submit(t+1) may precede collect(t).  The host reads back only detections, embeddings and the RLE strings; the masks
never leave the device.  results.mots_frame_result is the host restatement the tests compare against.

UnicornMOTSTracker is the n_seq = 1 case under the reference's one-sequence protocol."""
import torch

from . import ops
from .engine import UnicornEngine
from .mot import UnicornMOTBatch
from .tracker._stream import assoc_stream


class MaskEncoder:
    """uc_mots_encode for one frame at a time, or uc_mots_encode_batched for the frames of a batch, with the buffers it needs: the
    order / emit rows are uploaded from pinned memory and the strings are read back into a pinned buffer.  When a call needs more
    chars than the buffers hold, they grow and the (idempotent) encode runs again.  k_max: instances per call (over all frames of a
    batch)."""

    def __init__(self, k_max, device, capacity=1 << 16):
        self.dev, self.k_max = torch.device(device), k_max
        self.h_order = torch.zeros(k_max, dtype=torch.int32).pin_memory()
        self.h_emit = torch.zeros(k_max, dtype=torch.uint8).pin_memory()
        self.d_order = torch.zeros(k_max, dtype=torch.int32, device=device)
        self.d_emit = torch.zeros(k_max, dtype=torch.uint8, device=device)
        self.d_offsets = torch.zeros(k_max + 1, dtype=torch.int64, device=device)
        self.h_offsets = torch.zeros(k_max + 1, dtype=torch.int64).pin_memory()
        self.ws, self.ws_hw = None, (0, 0)
        self._alloc(capacity)

    def _alloc(self, capacity):
        self.d_chars = torch.empty(capacity, dtype=torch.uint8, device=self.dev)
        self.h_chars = torch.empty(capacity, dtype=torch.uint8).pin_memory()

    def _run(self, order, emit, img_h, img_w, encode):
        """Uploads the k = len(order) rows, runs encode(order, emit) (device views) on the current stream until the chars fit, and
        waits for the k strings."""
        k = len(order)
        assert 0 < k <= self.k_max
        self.reserve(img_h, img_w)
        self.h_order[:k] = torch.as_tensor(order, dtype=torch.int32)
        self.h_emit[:k] = torch.as_tensor(emit, dtype=torch.uint8)
        self.d_order[:k].copy_(self.h_order[:k], non_blocking=True)
        self.d_emit[:k].copy_(self.h_emit[:k], non_blocking=True)
        run = lambda: encode(self.d_order[:k], self.d_emit[:k])  # noqa: E731
        self.enqueue(k, run)
        return self.strings(k, run)

    def reserve(self, img_h, img_w):
        """Grows the workspace to k_max instances on an img_h x img_w frame."""
        if self.ws is None or img_h > self.ws_hw[0] or img_w > self.ws_hw[1]:
            self.ws_hw = (max(img_h, self.ws_hw[0]), max(img_w, self.ws_hw[1]))
            self.ws = ops.mots_encode_workspace(self.k_max, *self.ws_hw, self.dev)

    def enqueue(self, k, encode):
        """Runs encode() (launches that leave k strings in d_chars / d_offsets) on the current stream and queues the copy of the
        offsets; strings() then waits for them."""
        encode()
        self.h_offsets[:k + 1].copy_(self.d_offsets[:k + 1], non_blocking=True)

    def strings(self, k, encode):
        """The k strings of the encode enqueue(k, encode) queued on the current stream: waits for it, re-runs encode() with larger
        buffers while the chars do not fit, and reads the chars back."""
        stream = torch.cuda.current_stream()
        while True:
            stream.synchronize()
            total = int(self.h_offsets[k])
            if total <= self.d_chars.numel():
                break
            self._alloc(max(total, 2 * self.d_chars.numel()))
            self.enqueue(k, encode)
        self.h_chars[:total].copy_(self.d_chars[:total], non_blocking=True)
        stream.synchronize()
        s = self.h_chars[:total].numpy().tobytes().decode("ascii")
        off = self.h_offsets[:k + 1].tolist()
        return [s[off[i]:off[i + 1]] for i in range(k)]

    def __call__(self, masks, order, emit, thr, r, img_h, img_w):
        """masks fp32 [n_max,Hin,Win] (device); order: mask rows in ascending track id, emit: bools (host sequences).  Runs on the
        current stream and waits for its result.  Returns the k strings ("" where emit is false)."""
        if len(order) == 0:
            return []
        return self._run(order, emit, img_h, img_w, lambda o, e: ops.mots_encode(masks, o, e, thr, r, img_h, img_w, self.ws, self.d_chars,
                                                                                   self.d_offsets))

    def batch(self, masks, thr, frames):
        """masks fp32 [B,n_max,Hin,Win] (device); frames: B entries (order, emit, r, img_h, img_w) as in __call__, None for an image
        with nothing to encode.  One upload, one encode and two host synchronises for the whole batch (one more encode and
        synchronise when the chars outgrow the buffers).  A batch of one frame takes the one-frame launch, whose strings are the same.
        Returns B lists of strings."""
        _, _, Hin, Win = masks.shape
        frames = [f if f is not None else ([], [], 1.0, Hin, Win) for f in frames]
        if len(frames) == 1:
            order, emit, r, img_h, img_w = frames[0]
            return [self(masks[0], order, emit, thr, r, img_h, img_w)]
        ks = [len(f[0]) for f in frames]
        if sum(ks) == 0:
            return [[] for _ in frames]
        order = [row for f in frames for row in f[0]]
        emit = [e for f in frames for e in f[1]]
        rs, hs, ws = [f[2] for f in frames], [f[3] for f in frames], [f[4] for f in frames]
        flat = self._run(order, emit, max(hs), max(ws), lambda o, e: ops.mots_encode(masks, o, e, thr, rs, hs, ws, self.ws, self.d_chars,
                                                                                       self.d_offsets, k=ks))
        starts = [sum(ks[:b]) for b in range(len(ks))]
        return [flat[s:s + k] for s, k in zip(starts, ks)]


def _mots_match(tracker, d, f, scale, score_thr, frame_id, min_box_area):
    """The host half of a MOTS frame before its encode: score filter and QuasiDenseEmbedTracker.match(return_index=True) on the NMS rows
    d [n,7] and their embeddings f [n,128] -> the tracked instances in ascending id order: (bboxes [m,5] in original-image coordinates,
    ids [m], mask rows [m], emit [m]: the min_box_area rule)."""
    if d.shape[0] == 0:  # outputs[0] is None: no tracking for this frame (mot_evaluator.py:803)
        return torch.zeros(0, 5), torch.zeros(0, dtype=torch.long), torch.zeros(0, dtype=torch.long), []
    scores = d[:, 4] * d[:, 5]
    keep = scores > score_thr
    boxes = torch.cat([d[keep, :4] / scale, scores[keep, None]], 1)
    ob, _, oid, idx = tracker.match(boxes, torch.ones(boxes.size(0)), f[keep], frame_id, return_index=True)
    rows = torch.nonzero(keep).flatten()[idx]  # the mask row of every matched box (masks[keep][indexs], :838-840)
    valid = oid > -1
    ob, oid, rows = ob[valid], oid[valid], rows[valid]
    srt = oid.sort()[1]  # ascending track id (:842-846)
    ob, oid, rows = ob[srt], oid[srt], rows[srt]
    emit = [(x2 - x1) * (y2 - y1) > min_box_area for x1, y1, x2, y2 in ob[:, :4].tolist()]
    return ob, oid, rows, emit


def _mots_result(frame_id, ids, emit, rles, img_h, img_w):
    """The write_results_mots() tuple of a frame: (frame_id, ids (1-based), cat_id, img_h, img_w, rles) of the emitted instances."""
    return (frame_id, [int(t) + 1 for t, e in zip(ids.tolist(), emit) if e], 2, img_h, img_w, [s for s, e in zip(rles, emit) if e])


class UnicornMOTSBatch(UnicornMOTBatch):
    """`n_seq` MOTS sequences in lock step: the QD arm of UnicornMOTBatch (same start / submit / collect protocol, CUDA graphs, idle and
    never-started slots) with the mask head in the step.  The device half at B = n_seq adds the controllers, the mask branch and the
    dynamic masks of every image's NMS rows, written into the parity slot's own mask buffer [n_seq, max_dets, H, W]; collect() runs
    each active sequence's association, then one batched encode of all their tracked instances.  Each sequence's results equal
    those of the same driver at n_seq = 1.

    submit(frames, img_sizes, active) takes the n_seq original (h, w) instead of letterbox scales; collect() returns n_seq
    write_results_mots() tuples (frame_id, ids (1-based), cat_id, img_h, img_w, rles), None for a slot not stepped."""

    _tag = "motsb"

    def __init__(self, engine: UnicornEngine, input_size, n_seq, conf=0.01, nms=0.7, score_thr=0.1, max_dets=64, mask_thres=0.3, d_rate=2,
                 min_box_area=100, use_graph=False):
        if not engine.cfg["mask"]:
            raise ValueError("UnicornMOTSBatch: MOTS needs a *_mask model")
        super().__init__(engine, input_size, n_seq, conf, nms, score_thr, max_dets, "qd", use_graph)
        self.mask_thres, self.d_rate, self.min_box_area = mask_thres, d_rate, min_box_area
        H, W = self.input_size
        up = 8 // d_rate
        self._scratch = torch.empty(n_seq * max_dets * (H // 8) * (W // 8) * (1 + up * up), dtype=torch.float32, device=engine.dev)
        self._image_of = torch.arange(n_seq, dtype=torch.int32, device=engine.dev)  # head image b reads mask-branch image b
        for c in self._ctxs:  # per parity slot, so that the encode of step t reads its own masks while step t + 1 runs
            c.masks = torch.zeros(n_seq, max_dets, H, W, dtype=torch.float32, device=engine.dev)
            c.img_hw = [None] * n_seq
        self._enc = MaskEncoder(n_seq * max_dets, engine.dev)
        self.last_tracked = [None] * n_seq

    # ------------------------------------------------------------------------------------------ device half
    def _frame(self, c):
        e, one = c.eng, self.n_seq == 1
        e.begin_frame()
        fpn, seq = e.backbone(c.img, tag=c.tag)
        out = e.head(fpn, None, "mot", with_masks=True)
        # one sequence: the one-image launches; it needs no gate (a step without an active sequence does not run)
        dets, cnt = ops.postprocess_device(out[0] if one else out, e.ncls, self.conf, self.nms, c.ws)
        mf, um = e.mask_branch(fpn)
        hw = [(t.shape[1], t.shape[2]) for t in e.dyn_levels]
        ops.dynamic_masks(mf, um, e.dyn_levels, hw, c.ws, self.max_dets, up_rate=8 // self.d_rate, d_rate=self.d_rate,
                          out=c.masks[0] if one else c.masks, scratch=self._scratch, image_of=None if one else self._image_of)
        self._qd(e, seq["feat"], dets, cnt, gate=None if one else c.active)
        c.last = dict(head=out, mask_feats=mf, up_masks=um, dyn=list(e.dyn_levels))

    def submit(self, frames, img_sizes, active=None):
        """frames: preprocessed fp32 [n_seq,3,H,W] or uint8 [n_seq,H,W,3], host or device; img_sizes: n_seq original (h, w); active:
        n_seq flags (default: every started slot).  Enqueues the step; returns immediately."""
        try:
            sizes = [(int(h), int(w)) for h, w in img_sizes]
        except (TypeError, ValueError):
            sizes = None
        if sizes is None or len(sizes) != self.n_seq or any(h < 1 or w < 1 for h, w in sizes):
            raise ValueError(f"UnicornMOTSBatch: img_sizes must be {self.n_seq} original (h, w) >= 1, got {img_sizes!r}")
        H, W = self.input_size
        super().submit(frames, [min(H / float(h), W / float(w)) for h, w in sizes], active)
        self._ctxs[(self._ring.submitted - 1) % len(self._ctxs)].img_hw = sizes

    # ------------------------------------------------------------------------------------------ host half
    def collect(self):
        """Association and mask encoding of the oldest submitted step: n_seq write_results_mots() tuples, None for a slot not stepped.
        last_dets[i] / last_feats[i] then hold the NMS rows / embeddings slot i's tracker was given, and last_tracked[i] {"masks": the
        masks of those rows (device), "boxes", "ids", "rows": the tracked boxes, their ids and mask rows in ascending id} (None for such
        a slot)."""
        c = self._ring.collect()
        c.event.synchronize()
        n_seq = self.n_seq
        self.last_dets, self.last_feats, self.last_tracked = [None] * n_seq, [None] * n_seq, [None] * n_seq
        tracked, frames = {}, [None] * n_seq
        for i in range(n_seq):
            if not c.mask[i]:
                continue
            n = min(int(c.host_count[i]), self.n_keep)
            d, f = c.host_dets[i, :n].clone(), c.host_feats[i, :n].clone()
            self.last_dets[i], self.last_feats[i] = d, f
            ob, oid, rows, emit = _mots_match(c.trackers[i], d, f, c.scales[i], self.score_thr, c.frame_ids[i], self.min_box_area)
            self.last_tracked[i] = dict(masks=c.masks[i, :n], boxes=ob, ids=oid, rows=rows)
            tracked[i] = oid, emit
            frames[i] = (rows.tolist(), emit, c.scales[i], *c.img_hw[i])
        stream = assoc_stream(self.eng.dev)
        with torch.cuda.stream(stream):  # not behind the next step's kernels on the main stream
            stream.wait_event(c.event)
            # the encoder waits for its strings, so the encode has read c.masks before collect() returns: submit(t + 2), which
            # rewrites this slot's mask buffer, is issued only after that
            rles = self._enc.batch(c.masks, self.mask_thres, frames)
        res = [None] * n_seq
        for i, (oid, emit) in tracked.items():
            res[i] = _mots_result(c.frame_ids[i], oid, emit, rles[i], *c.img_hw[i])
        return res

    def step_tensor(self, frames, img_sizes, active=None):
        """Sequential protocol: one step in, its n_seq results out."""
        self.submit(frames, img_sizes, active)
        return self.collect()


class UnicornMOTSTracker:
    """One MOTS sequence: UnicornMOTSBatch at n_seq = 1 (same arguments) with its slot started on `tracker` (default a fresh
    QuasiDenseEmbedTracker), under the reference's one-sequence protocol.  last: the device tensors of the latest submitted frame
    (head, mask_feats, up_masks, dyn) and, from the latest collect(), the NMS rows / embeddings the tracker was given (dets, feats),
    the rows' masks (masks) and the tracked boxes, ids and mask rows in ascending id (boxes, ids, rows)."""

    def __init__(self, engine: UnicornEngine, input_size, conf=0.01, nms=0.7, score_thr=0.1, max_dets=64, mask_thres=0.3, d_rate=2,
                 min_box_area=100, tracker=None, use_graph=False):
        self._b = UnicornMOTSBatch(engine, input_size, 1, conf, nms, score_thr, max_dets, mask_thres, d_rate, min_box_area, use_graph)
        self._b.start(0, tracker)
        self.tracker = self._b.trackers[0]

    max_dets = property(lambda self: self._b.max_dets)
    mask_thres = property(lambda self: self._b.mask_thres)
    min_box_area = property(lambda self: self._b.min_box_area)
    _ctxs = property(lambda self: self._b._ctxs)
    frame_id = property(lambda self: self._b.frame_ids[0])  # frames submitted
    last = property(lambda self: self._b.last)

    def submit(self, frame, img_h, img_w):
        """frame: preprocessed fp32 [1,3,H,W] or uint8 [1,H,W,3], host or device; (img_h, img_w): original image size.  Enqueues
        the frame; returns immediately."""
        self._b.submit(frame, [(img_h, img_w)])

    def collect(self):
        """Association and mask encoding of the oldest submitted frame.  Returns the tuple write_results_mots() consumes:
        (frame_id, ids (1-based), cat_id, img_h, img_w, rles)."""
        res = self._b.collect()[0]
        self.last.update(dets=self._b.last_dets[0], feats=self._b.last_feats[0], **self._b.last_tracked[0])
        return res

    def step_tensor(self, frame, img_h, img_w):
        """Sequential protocol of the reference: one frame in, its write_results_mots() tuple out."""
        self.submit(frame, img_h, img_w)
        return self.collect()

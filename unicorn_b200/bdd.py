"""BDD100K MOT and MOTS under qdtrack's test protocol (external/qdtrack/qdtrack/apis/test_omni.py, multi_gpu_test_omni), batched over
`n_seq` sequences like UnicornMOTBatch (mot.py).  It differs from evaluate_omni (mot.py / mots.py) as follows:

  - the tracker gets each detection's class (the NMS class column) and matches within a class (with_cats);
  - there is no score filter: every NMS row is associated;
  - the tracker settings are qdtrack's BDD100K configs (tracker.bdd_tracker);
  - pre_dict is set by a sequence's first step whether or not it had detections (test_omni.py:97-98), then advances only on steps
    with detections: QDEmbedding(first_step=True), still a device-side update inside the step's graph;
  - frame ids are 0-based (mmdet's frame_id);
  - MOTS encodes the mask of EVERY detection, class-wise and without overlap removal, and the tracked instances take the same
    strings: the NMS-order rows at the positions where the tracker's score-ordered duplicate mask (`valids`) is true, then the
    ids > -1 (test_omni.py:139-147, literally);
  - each frame's result is test_omni's dict, built by results.bbox2result / track2result / segtrack2result.

Frames come letterboxed (top-left, pad 114) as for UnicornMOTSBatch.  BDD100K frames are 720x1280, so at 800x1280 r = 1 and the
mmdet test pipeline plus test_omni.preprocess reduce to that letterbox.  At other ratios they are not equivalent: the reference
resizes float pixels with cv2 and truncates to uint8."""
import warnings
from collections import defaultdict

import numpy as np
import torch

from . import ops
from .det import RowMasks
from .frames import anchor_count
from .mot import UnicornMOTBatch
from .results import bbox2result, rle_dict, segtrack2result, track2result
from .tracker import bdd_tracker
from .tracker._stream import assoc_stream


def _det_bboxes(d, scale):
    """test_omni.py:103-127: NMS rows d [n, 7] -> (det_bboxes [n, 5] = boxes / scale and obj * cls, labels [n])."""
    return torch.cat([d[:, :4] / scale, d[:, 4:5] * d[:, 5:6]], 1), d[:, 6].clone()


def bdd_mot_result(tracker, d, f, scale, frame_id, num_classes):
    """One frame of test_omni.py's MOT branch on the NMS rows d [n, 7] and their embeddings f [n, 128]: dict(bbox_results,
    track_results)."""
    if d.shape[0] == 0:  # outputs[0] is None (:178-181): the tracker is not called
        return dict(bbox_results=bbox2result(np.zeros((0, 5)), None, num_classes),
                    track_results=[np.zeros((0, 6), dtype=np.float32) for _ in range(num_classes)])
    det_bboxes, labels = _det_bboxes(d, scale)
    tb, tl, ids = tracker.match(det_bboxes, labels, f, frame_id)
    return dict(bbox_results=bbox2result(det_bboxes, labels, num_classes), track_results=track2result(tb, tl, ids, num_classes))


def bdd_mots_result(tracker, d, f, scale, frame_id, rles, img_h, img_w, num_classes):
    """One frame of test_omni.py's MOTS branch: rles[n] is the RLE string of NMS row n's mask over img_h x img_w.  Returns
    {"track_result", "bbox_result", "segm_result"}."""
    if d.shape[0] == 0:  # :173-177
        return {"track_result": defaultdict(list), "bbox_result": bbox2result(np.zeros((0, 5)), None, num_classes),
                "segm_result": [[] for _ in range(num_classes)]}
    det_bboxes, labels = _det_bboxes(d, scale)
    tb, tl, ids, valids = tracker.match(det_bboxes, labels, f, frame_id, return_index=True)
    segms = [rle_dict(rles[r], img_h, img_w) for r in torch.nonzero(valids).flatten().tolist()]  # masks_full[indexs] (:145)
    segm_result = [[] for _ in range(num_classes)]
    for n, label in enumerate(labels.tolist()):
        segm_result[int(label)].append(rle_dict(rles[n], img_h, img_w))
    return {"track_result": segtrack2result(tb, tl, segms, ids), "bbox_result": bbox2result(det_bboxes, labels, num_classes),
            "segm_result": segm_result}


class UnicornBDDMOTBatch(UnicornMOTBatch):
    """test_omni.py's MOT branch for `n_seq` sequences in lock step: UnicornMOTBatch's QD arm (device half, CUDA graphs, two parity
    slots, start / submit / collect, idle slots) under the BDD100K protocol (module docstring).  Serves the plain tracking configs; a
    `*_mask` checkpoint loads into them with load_checkpoint(..., strict=False), as the reference's BDD100K recipe does.

    start(i, tracker=None) begins a sequence in slot i (default: bdd_tracker()).  submit(frames, img_sizes, active): letterboxed
    frames and the n_seq original (h, w).  collect(): per sequence the frame's dict(bbox_results, track_results), None for an idle
    slot.

    max_dets: the rows per sequence and step that are read back and associated (MOTS: encoded too).  The reference has no cap, so the
    lowest rows beyond it are dropped with a warning; the default 4096 is above the ~2900 rows per frame seeded weights leave at conf
    0.01 and 800x1280 (DESIGN.md section 4.13), and max_dets=None reads back one row per anchor, so that nothing can be dropped."""

    _tag = "bdd"
    _first_step = True
    _mots = False

    def __init__(self, engine, input_size=(800, 1280), n_seq=1, conf=0.01, nms=0.65, max_dets=4096, use_graph=True):
        H, W = input_size
        super().__init__(engine, input_size, n_seq, conf, nms, None, anchor_count(H, W) if max_dets is None else max_dets, "qd", use_graph)
        self.num_classes = engine.ncls
        for c in self._ctxs:
            c.img_hw = [None] * n_seq

    def start(self, i, tracker=None):
        """Begin a new sequence in slot i with `tracker` (default: the BDD100K settings); its frame ids restart at 0."""
        super().start(i, tracker if tracker is not None else bdd_tracker(self._mots, self.eng.dev))

    def submit(self, frames, img_sizes, active=None):
        """frames: letterboxed fp32 [n_seq,3,H,W] or uint8 [n_seq,H,W,3], host or device; img_sizes: n_seq original (h, w); active:
        n_seq flags (default: every started slot).  Enqueues the step; returns immediately."""
        try:
            sizes = [(int(h), int(w)) for h, w in img_sizes]
        except (TypeError, ValueError):
            sizes = None
        if sizes is None or len(sizes) != self.n_seq or any(h < 1 or w < 1 for h, w in sizes):
            raise ValueError(f"{type(self).__name__}: img_sizes must be {self.n_seq} original (h, w) >= 1, got {img_sizes!r}")
        H, W = self.input_size
        super().submit(frames, [min(H / float(h), W / float(w)) for h, w in sizes], active)  # test_omni.py:122
        self._ctxs[(self._ring.submitted - 1) % len(self._ctxs)].img_hw = sizes

    def _rows(self, c, i):
        """Sequence i's NMS rows and embeddings of the collected step c."""
        total = int(c.host_count[i])
        if total > self.max_dets and not self._warned:
            warnings.warn(f"{type(self).__name__}: {total} detections after NMS in slot {i}, only the {self.max_dets} best are "
                          "associated (raise max_dets; the reference has no cap)")
            self._warned = True
        k = min(total, self.n_keep)
        self.last_dets[i], self.last_feats[i] = c.host_dets[i, :k].clone(), c.host_feats[i, :k].clone()
        return self.last_dets[i], self.last_feats[i]

    def collect(self):
        """The oldest submitted step's per-frame dicts (test_omni.py's MOT branch), None for a slot not stepped."""
        c = self._ring.collect()
        c.event.synchronize()
        res = [None] * self.n_seq
        self.last_dets, self.last_feats = [None] * self.n_seq, [None] * self.n_seq
        for i in range(self.n_seq):
            if c.mask[i]:
                d, f = self._rows(c, i)
                res[i] = bdd_mot_result(c.trackers[i], d, f, c.scales[i], c.frame_ids[i] - 1, self.num_classes)
        return res

    def step_tensor(self, frames, img_sizes, active=None):
        """Sequential protocol: one step in, its n_seq results out."""
        self.submit(frames, img_sizes, active)
        return self.collect()


class UnicornBDDMOTSBatch(UnicornBDDMOTBatch):
    """test_omni.py's MOTS branch for `n_seq` sequences of a `*_mask` config: the frame of UnicornBDDMOTBatch with the controllers and
    the mask branch, and the mask of every NMS row of every sequence encoded to COCO RLE over the sequence's own original frame,
    `chunk` rows at a time (det.RowMasks, the chunk loop of UnicornInstanceSegmenter).  The graph ends with the masks of rows
    [0, chunk); collect() encodes them and any further chunks on the association stream, so the next step's device work overlaps.

    collect(): per sequence {"track_result", "bbox_result", "segm_result"} with RLE dicts {"size": [h, w], "counts": bytes}, None
    for an idle slot.  The parity slots run on two engine contexts (UnicornEngine.fork) with their own NMS workspaces, so the step
    in flight does not overwrite the mask inputs and NMS rows a later chunk of the collected step reads."""

    _tag = "bddm"
    _mots = True
    _with_masks = True

    def __init__(self, engine, input_size=(800, 1280), n_seq=1, conf=0.01, nms=0.65, mask_thres=0.3, d_rate=2, chunk=100, max_dets=4096,
                 use_graph=True, capacity=1 << 20):
        if not engine.cfg["mask"]:
            raise ValueError(f"UnicornBDDMOTSBatch: MOTS needs a *_mask model, got {engine.cfg_name}")
        if d_rate != 2 or chunk < 1 or n_seq > 64 or n_seq * chunk > 65535:
            raise ValueError(f"UnicornBDDMOTSBatch: d_rate 2 (the 144-channel up-mask layer upsamples x4), chunk >= 1, n_seq <= 64 and "
                             f"n_seq * chunk <= 65535 (got {d_rate}, {chunk}, {n_seq})")
        super().__init__(engine, input_size, n_seq, conf, nms, max_dets, use_graph)
        self.mask_thres, self.d_rate, self.chunk = mask_thres, d_rate, chunk
        H, W = self.input_size
        A = anchor_count(H, W)
        slot1 = self._ctxs[1]
        slot1.eng, slot1.ws = engine.fork(), ops.PostWorkspace(A, engine.dev, n_seq)
        for c in self._ctxs:
            c.rows = RowMasks(n_seq, A, self.input_size, chunk, d_rate, mask_thres, engine.dev, capacity)

    def _after_nms(self, c, fpn):
        c.mf, c.um = c.eng.mask_branch(fpn)
        c.dyn = list(c.eng.dyn_levels)
        c.rows.masks(c.mf, c.um, c.dyn, c.ws, 0)

    def collect(self):
        """The oldest submitted step's per-frame dicts (test_omni.py's MOTS branch), None for a slot not stepped."""
        c = self._ring.collect()
        c.event.synchronize()
        n = self.n_seq
        res = [None] * n
        self.last_dets, self.last_feats, self.last_rles = [None] * n, [None] * n, [None] * n
        rows = [self._rows(c, i) if c.mask[i] else None for i in range(n)]
        counts = [r[0].shape[0] if r is not None else 0 for r in rows]
        sizes = [hw if hw is not None else self.input_size for hw in c.img_hw]
        if not any(c.mask):  # nothing ran
            return res
        stream = assoc_stream(self.eng.dev)
        with torch.cuda.stream(stream):  # not behind the next step's kernels on the main stream
            stream.wait_event(c.event)
            if n > 1:
                c.ws.count.mul_(c.active)  # an idle sequence's rows (of a stale frame) are not encoded
            c.rows.enqueue(n, c.ws, c.scales, sizes)
            rles = c.rows.strings(counts, c.mf, c.um, c.dyn, c.ws, c.scales, sizes)
        for i in range(n):
            if c.mask[i]:
                self.last_rles[i] = rles[i]
                res[i] = bdd_mots_result(c.trackers[i], *rows[i], c.scales[i], c.frame_ids[i] - 1, rles[i], *c.img_hw[i], self.num_classes)
        return res

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
resizes float pixels with cv2 and truncates to uint8.

BDDBitmasks and write_seg_track take the MOTS track_result dicts on to qdtrack's seg_track format (tools/to_bdd100k.py --task
seg_track: core/to_bdd100k/transforms.py seg_track_to_bdd100k and utils.py mask_prepare / mask_merge), one RGBA "bitmask" PNG per
frame, with the masks decoded and painted on the device (uc_bdd_bitmask_batched)."""
import os
import warnings
from collections import defaultdict

import numpy as np
import torch

from . import ops, post_ops
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


BDD_MAX_FRAMES = 64  # UC_MOTS_MAX_IMAGES: frames per uc_bdd_bitmask_batched call
_BAD = ((post_ops.BDD_BAD_CHARS, "bad chars"), (post_ops.BDD_BAD_RUNS, "runs that do not cover the frame"),
        (post_ops.BDD_BAD_INDEX, "bad offsets or paint order"))


def _channel(v):
    """What mask_merge stores in a channel where the mask is 1: bitmask * (1 - m) + m * v with m uint8, cast back to uint8 (a float
    value is truncated, an integer one wraps).  v: one value per instance."""
    return (np.ones(len(v), np.uint8) * v).astype(np.uint8)


def _frame(track_dict, h, w, f):
    """mask_prepare (utils.py:15-22) of one frame without the decode: its strings, packed colours (uint32, R in the low byte) and
    paint ranks."""
    strings, labels, scores = [], [], []
    for id_, inst in track_dict.items():
        segm = inst["segm"]
        if [int(v) for v in segm["size"]] != [h, w]:
            raise ValueError(f"BDDBitmasks: frame {f}, track {id_}: segm size {list(segm['size'])} is not the frame's [{h}, {w}]")
        c = segm["counts"]
        strings.append(c.encode("ascii") if isinstance(c, str) else bytes(c))
        labels.append(inst["label"])
        scores.append(inst["bbox"][-1])
    r = np.array(labels) + 1  # segtrack2result's labels are float32: so is label + 1
    if not (np.isfinite(r) & (r >= 0) & (r < 256)).all():
        raise ValueError(f"BDDBitmasks: frame {f}: label + 1 = {r[~(np.isfinite(r) & (r >= 0) & (r < 256))][0]} does not fit a uint8 channel")
    ids = np.array(list(track_dict), dtype=np.int64)  # segtrack2result's keys are int64
    rgba = np.stack([_channel(r), np.zeros(len(ids), np.uint8), _channel(ids >> 8), _channel(ids & 255)], 1)
    ranks = np.empty(len(strings), dtype=np.int32)
    ranks[np.argsort(scores)] = np.arange(len(strings), dtype=np.int32)  # the reference's own sort: ties as numpy orders them
    return strings, np.ascontiguousarray(rgba).view("<u4").reshape(-1), ranks


class BDDBitmasks:
    """qdtrack's seg_track bitmasks of up to BDD_MAX_FRAMES frames per call on `device`: paint(track_results, sizes) packs every
    frame's strings, colours and paint order (np.argsort of the scores, as mask_merge) on the host, uploads them in one copy and runs
    one uc_bdd_bitmask_batched.  The pinned and device buffers grow on demand.  A bitmask has its frame's original size; the reference
    hard-codes 720 x 1280, the BDD100K size."""

    def __init__(self, device="cuda", capacity=1 << 16):
        self.dev, self.capacity = torch.device(device), capacity
        self._h_in = self._d_in = self._out = self._h_out = self._ws = None  # allocated by the first paint()
        self._status = self._h_status = None

    def _grow(self, t, n, pinned=False):
        """t, or a larger buffer (pinned host or on the device) when t holds fewer than n bytes."""
        if t is not None and t.numel() >= n:
            return t
        n = max(n, 2 * t.numel() if t is not None else self.capacity)
        return torch.empty(n, dtype=torch.uint8).pin_memory() if pinned else torch.empty(n, dtype=torch.uint8, device=self.dev)

    def paint(self, track_results, sizes, host=False):
        """track_results: 1..64 track_result dicts ({id: {"bbox", "label", "segm"}}, as UnicornBDDMOTSBatch.collect() returns them or
        as loaded from a results pickle), sizes: each frame's original (h, w); every segm["size"] must equal it.  Returns the uint8
        [h, w, 4] bitmasks, device views valid until the next call (host=True: numpy views of pinned memory).  A malformed RLE string
        raises ValueError."""
        B = len(track_results)
        if not 1 <= B <= BDD_MAX_FRAMES or len(sizes) != B:
            raise ValueError(f"BDDBitmasks.paint: 1..{BDD_MAX_FRAMES} frames with one (h, w) each, got {B} frames, {len(sizes)} sizes")
        hs, ws = [int(s[0]) for s in sizes], [int(s[1]) for s in sizes]
        if any(h < 1 or w < 1 for h, w in zip(hs, ws)):
            raise ValueError(f"BDDBitmasks.paint: bad frame sizes {list(sizes)}")
        strings, colors, ranks, k = [], [], [], []
        for f, (d, h, w) in enumerate(zip(track_results, hs, ws)):
            s, c, r = _frame(d, h, w, f)
            strings += s
            colors.append(c)
            ranks.append(r)
            k.append(len(s))
        K = len(strings)
        chars = b"".join(strings)
        offsets = np.zeros(K + 1, dtype=np.int64)
        np.cumsum([len(s) for s in strings], out=offsets[1:])
        # one upload: offsets | colours | ranks | chars, each 16-byte aligned
        o_col = (8 * (K + 1) + 15) & ~15
        o_rank = o_col + ((4 * K + 15) & ~15)
        o_chars = o_rank + ((4 * K + 15) & ~15)
        total = o_chars + max(len(chars), 1)
        self._h_in = self._grow(self._h_in, total, pinned=True)
        self._d_in = self._grow(self._d_in, total)
        h = self._h_in.numpy()
        h[:8 * (K + 1)] = offsets.view(np.uint8)
        h[o_col:o_col + 4 * K] = np.concatenate(colors).view(np.uint8)
        h[o_rank:o_rank + 4 * K] = np.concatenate(ranks + [np.zeros(0, np.int32)]).view(np.uint8)
        h[o_chars:o_chars + len(chars)] = np.frombuffer(chars, dtype=np.uint8)
        with torch.cuda.device(self.dev):
            out = self._launch(total, K, o_col, o_rank, o_chars, len(chars), k, hs, ws, host)
        bad = [(f, int(v)) for f, v in enumerate(self._h_status[:B].tolist()) if v]
        if bad:
            raise ValueError("BDDBitmasks.paint: malformed segm RLE: " + "; ".join(
                f"frame {f}: " + ", ".join(what for bit, what in _BAD if v & bit) for f, v in bad))
        return out

    def _launch(self, total, K, o_col, o_rank, o_chars, n_chars, k, hs, ws, host):
        """Uploads the packed inputs, paints, reads back the status (and with host=True the bitmasks) and waits."""
        B = len(k)
        if self._status is None:
            self._status = torch.zeros(BDD_MAX_FRAMES, dtype=torch.int32, device=self.dev)
            self._h_status = torch.zeros(BDD_MAX_FRAMES, dtype=torch.int32).pin_memory()
        d = self._d_in
        d[:total].copy_(self._h_in[:total], non_blocking=True)
        out_off = np.zeros(B + 1, dtype=np.int64)
        np.cumsum([4 * h * w for h, w in zip(hs, ws)], out=out_off[1:])
        self._out = self._grow(self._out, int(out_off[B]))
        self._ws = self._grow(self._ws, post_ops.bdd_bitmask_workspace_bytes(k, hs, ws, n_chars))
        n = 4 * max(K, 1)  # not empty: an empty view has no data pointer (nothing is read for K = 0)
        post_ops.bdd_bitmask(d[o_chars:], n_chars, d[:8 * (K + 1)].view(torch.int64), d[o_col:o_col + n].view(torch.int32),
                             d[o_rank:o_rank + n].view(torch.int32), k, hs, ws, self._out, out_off[:B].tolist(), self._ws, self._status)
        out = self._out
        self._h_status[:B].copy_(self._status[:B], non_blocking=True)
        if host:
            self._h_out = self._grow(self._h_out, int(out_off[B]), pinned=True)
            self._h_out[:int(out_off[B])].copy_(self._out[:int(out_off[B])], non_blocking=True)
            out = self._h_out
        torch.cuda.current_stream().synchronize()
        views = [out[int(out_off[f]):int(out_off[f + 1])].view(hs[f], ws[f], 4) for f in range(B)]
        return [v.numpy() for v in views] if host else views


def write_seg_track(track_results, img_names, out_base, sizes, painter=None, batch=BDD_MAX_FRAMES):
    """qdtrack's seg_track_to_bdd100k (core/to_bdd100k/transforms.py): frame i's bitmask as an RGBA PNG at
    out_base/seg_track/<img_names[i] with .jpg replaced by .png>, written with PIL as mask_merge does.  track_results, img_names and
    sizes ((h, w) per frame) run in parallel; the bitmasks are painted `batch` frames per call.  Returns the paths written."""
    from PIL import Image
    if not len(track_results) == len(img_names) == len(sizes):
        raise ValueError("write_seg_track: track_results, img_names and sizes must have one entry per frame")
    painter = painter or BDDBitmasks()
    base = os.path.join(out_base, "seg_track")
    os.makedirs(base, exist_ok=True)
    paths = []
    for i in range(0, len(track_results), batch):
        for name, bm in zip(img_names[i:i + batch], painter.paint(track_results[i:i + batch], sizes[i:i + batch], host=True)):
            path = os.path.join(base, name.replace(".jpg", ".png"))
            os.makedirs(os.path.dirname(path), exist_ok=True)
            Image.fromarray(bm).save(path)
            paths.append(path)
    return paths

"""VOS per-frame driver on the H100 engine — mirrors external/lib/test/tracker/unicorn_vos.py: `initialize` :43-69, `track`
:71-127 (objects of the first frame, reference groups of objects that appear later :79-84, :86-98, soft aggregation + argmax
:105-121), `get_mask_results` :129-155 (best instance per object, mask resized to the original frame), `get_det_results`
:157-201 (interaction, correlation, per-object prior pyramid -> mask head -> postprocess_inst).

H100 restructuring, same results: one backbone pass and one mask-branch pass per frame (the reference recomputes the mask branch
inside the head for every object); per reference group ONE fused correlation launch propagates the label maps of all its
objects (the 16000^2 similarity matrix never exists); the resize to the original frame, the float32 background product and the
argmax run in one kernel on the device (uc_vos_aggregate); the only per-frame host traffic is the frame in, the label map and the
detection rows out.  With use_graph=True the steady-state frame is one CUDA-graph replay (re-captured when objects are added).

depth > 1: like in SOT, a frame depends only on the reference frames of its objects, never on the previous frame's result, so
`submit(frame)` / `collect()` keep `depth` steady-state frames in flight, each in its own frame slot (engine fork, stream, buffers)
sharing the reference groups; frames that add objects go through track_tensor() on slot 0 with the pipeline drained.
"""
import torch

from . import ops
from .engine import UnicornEngine
from .frames import FrameSlot, Ring, anchor_count, in_flight
from .sot import LetterboxBatch, get_label_map, letterbox_frame, state_xywh, xyxy_resized


def label_values(boxes_xyxy, input_size, device):
    """The stride-8 label values of each box (unicorn_vos.py:66-69, get_label_map at 1/8 resolution): fp32 [len(boxes), H/8*W/8]."""
    H, W = input_size
    maps = [ops.bilinear(get_label_map(b, H, W, device), H // 8, W // 8, 8.0, 8.0).reshape(1, -1) for b in boxes_xyxy]
    return torch.cat(maps, 0).contiguous()


class _Group:
    """Objects sharing one reference frame (unicorn_vos.py: out_dict_pre / out_dict_pre_new[i])."""

    def __init__(self, ref_feat, ref_proj, obj_ids, lbs):
        self.ref_feat, self.ref_proj, self.obj_ids, self.lbs = ref_feat, ref_proj, list(obj_ids), lbs


class _Slot(FrameSlot):
    """One VOS frame in flight: a frame slot plus the per-object mask and detection buffers, the label map and soft masks at the
    original resolution, the pinned detection rows and the group sizes its graph was captured for."""

    def __init__(self, eng, H, W, stream):
        super().__init__(eng, H, W, stream)
        self.mask_bufs, self.det_bufs = [], []  # per object: fp32 [1,H,W] best-instance mask, fp32 [8] = det row + count
        self.seg = self.soft = self.rows_host = self.graph_key = None
        self.frames = 0  # since initialize_tensor: the first one runs eagerly

    # bench.py reads vos._workers[i]._stream / ._graph
    _stream = property(lambda self: self.stream)
    _graph = property(lambda self: self.graph)


class UnicornVOSTrack:
    def __init__(self, engine: UnicornEngine, input_size, conf=0.001, nms=0.65, max_inst=1, d_rate=2, use_graph=False, depth=1):
        assert engine.cfg["mask"], "VOS needs a *_mask model"
        assert depth >= 1
        self.eng, self.input_size = engine, tuple(input_size)
        self.conf, self.nms, self.max_inst, self.d_rate = conf, nms, max_inst, d_rate
        self.num_classes = 1
        H, W = self.input_size
        self.use_graph = use_graph
        self.groups = []
        self.state_pre_dict = {}
        self.debug = False  # tests: keep per-object copies of the head output and the controller maps
        self.launches_per_frame = 0  # bench.py reads it
        self.depth = depth
        self._ring = Ring(in_flight(engine, depth, lambda eng, stream: _Slot(eng, H, W, stream)))
        self._workers = self._ring.slots  # bench.py reads vos._workers[i]

    # slot 0 runs initialize_tensor() and track_tensor() (tests read these)
    last = property(lambda self: self._workers[0].last)
    _soft = property(lambda self: self._workers[0].soft)

    # ------------------------------------------------------------------------------------------ helpers
    def _label_maps(self, boxes_xyxy):
        return label_values(boxes_xyxy, self.input_size, self.eng.dev)

    def _obj_bufs(self, s, i):
        H, W = self.input_size
        while len(s.mask_bufs) <= i:
            s.mask_bufs.append(torch.zeros(1, H, W, dtype=torch.float32, device=self.eng.dev))
            s.det_bufs.append(torch.zeros(8, dtype=torch.float32, device=self.eng.dev))
        return s.mask_bufs[i], s.det_bufs[i]

    @property
    def obj_ids(self):
        return [o for g in self.groups for o in g.obj_ids]

    # ------------------------------------------------------------------------------------------ tensor protocol
    def initialize_tensor(self, ref_frame, boxes_xyxy, orig_size=None, r=1.0):
        """ref_frame: preprocessed fp32 [1,3,H,W] or uint8 [1,H,W,3]; boxes_xyxy: dict obj_id -> box in resized-image coordinates
        (unicorn_vos.py:60-66); orig_size = (height, width) of the original frames (default: the network input size), r = resize
        ratio of the letterbox."""
        e = self.eng
        inp = self._workers[0].stage(ref_frame)
        e.begin_frame()
        _, seq = e.backbone(inp, tag="ref")
        ids = list(boxes_xyxy.keys())
        ref_feat = seq["feat"].clone()
        self.groups = [_Group(ref_feat, e.project_ref(ref_feat), ids, self._label_maps([boxes_xyxy[o] for o in ids]))]
        self.orig_size = tuple(orig_size) if orig_size is not None else self.input_size
        self.r = float(r)
        self._ring.reset()
        for s in self._workers:
            s.frames = 0
        torch.cuda.synchronize()

    def _device_frame(self, s):
        """Every kernel of one steady-state frame in slot s (no host synchronisation; CUDA-graph capturable)."""
        e = s.eng
        H, W = self.input_size
        hh, ww = H // 8, W // 8
        e.begin_frame()
        fpn, seq = e.backbone(s.img, tag="cur")
        mf, um = e.mask_branch(fpn)  # identical for every object: computed once per frame
        s.last = dict(mask_feats=mf, up_masks=um, per_obj={}, feat=seq["feat"], coarse={})
        slot = 0
        for gi, g in enumerate(self.groups):
            f_pre, f_cur = e.interaction(g.ref_feat, seq["feat"], ref_proj=g.ref_proj)
            e_pre, e_cur = e.upsample(f_pre, "embp"), e.upsample(f_cur, "embc")
            K = len(g.obj_ids)
            for c0 in range(0, K, 8):  # uc_corr_propagate carries up to 8 value rows per launch
                kc = min(8, K - c0)
                coarse = ops.corr_propagate(e_pre.view(-1, 128), e_cur.view(-1, 128), g.lbs[c0:c0 + kc],
                                            out=e.buf(f"vos.coarse{gi}.{c0}", (kc, hh * ww), torch.float32))
                for i in range(kc):
                    oid = g.obj_ids[c0 + i]
                    c = coarse[i:i + 1].view(1, hh, ww)
                    pri = (c, ops.bilinear(c, hh // 2, ww // 2, 2.0, 2.0, out=e.buf("vos.p1", (1, hh // 2, ww // 2), torch.float32)),
                           ops.bilinear(c, hh // 4, ww // 4, 4.0, 4.0, out=e.buf("vos.p2", (1, hh // 4, ww // 4), torch.float32)))
                    head = e.head(fpn, pri, "sot", with_masks=True)
                    ops.postprocess_device(head[0], 1, self.conf, self.nms, s.ws, max_keep=self.max_inst)
                    mask, det = self._obj_bufs(s, slot)
                    mask.zero_()  # an object without a detection contributes an all-zero mask (unicorn_vos.py:154-155)
                    hw = [(t.shape[1], t.shape[2]) for t in e.dyn_levels]
                    up = 8 // self.d_rate
                    ops.dynamic_masks(mf, um, e.dyn_levels, hw, s.ws, 1, up_rate=up, d_rate=self.d_rate, out=mask,
                                      scratch=e.buf("vos.scratch", (hh * ww * (1 + up * up),), torch.float32))
                    det[:7].copy_(s.ws.dets[0])
                    det[7:8].copy_(s.ws.count.view(1).float())
                    keep = (lambda t: t.clone()) if self.debug else (lambda t: t)
                    s.last["per_obj"][oid] = dict(head=keep(head), dyn=[keep(t) for t in e.dyn_levels], slot=slot)
                    s.last["coarse"][oid] = c
                    slot += 1
        return seq

    def _aggregate(self, s, new_ids=(), init_mask=None):
        """unicorn_vos.py:100-127 on the device, into s.seg (segmentation uint8 [H0,W0]) and s.soft (soft masks fp32 [n,H0,W0])."""
        H, W = self.input_size
        H0, W0 = self.orig_size
        ids = self.obj_ids + list(new_ids)
        n = len(ids)
        if s.seg is None or s.seg.shape != (H0, W0) or s.soft.shape[0] < n:
            s.seg = torch.zeros(H0, W0, dtype=torch.uint8, device=self.eng.dev)
            s.soft = torch.zeros(max(n, 4), H0, W0, dtype=torch.float32, device=self.eng.dev)
        ops.vos_aggregate(s.mask_bufs[:len(self.obj_ids)], init_mask, ids, H, W, self.r, s.soft, s.seg)

    def _enqueue(self, s, cur_frame, new_ids=(), new_boxes_xyxy=None, init_mask=None):
        """Device half of a frame in slot s on the current stream + the asynchronous read of the detection rows; no host
        synchronisation unless a graph has to be (re)captured."""
        s.frames += 1
        s.stage(cur_frame)
        key = tuple(len(g.obj_ids) for g in self.groups)
        if self.use_graph and not new_ids and s.frames > 1:
            if s.graph is None or s.graph_key != key:
                s.graph, self.launches_per_frame = s.capture(lambda: (self._device_frame(s), self._aggregate(s)), warmup=True)
                s.graph_key = key
            else:
                s.graph.replay()
        else:
            seq = self._device_frame(s)
            self._aggregate(s, new_ids, init_mask)
            if new_ids:  # this frame becomes the reference of the new objects (unicorn_vos.py:87-88)
                ref_feat = seq["feat"].clone()
                self.groups.append(_Group(ref_feat, self.eng.project_ref(ref_feat), new_ids, self._label_maps([new_boxes_xyxy[o] for o in new_ids])))
                s.graph = None
        n_old = len(s.last["per_obj"])
        if n_old:  # one D2H read: detection rows + counts, into pinned memory
            if s.rows_host is None or s.rows_host.shape[0] < n_old:
                s.rows_host = torch.zeros(max(n_old, 4), 8).pin_memory()
            s.rows_host[:n_old].copy_(torch.stack(s.det_bufs[:n_old]), non_blocking=True)
        s.event.record()

    def _finish(self, s):
        """Result of the frame enqueued in slot s (objects are only added with no frame in flight, so obj_ids are the frame's)."""
        n_old = len(s.last["per_obj"])
        s.event.synchronize()
        rows = s.rows_host[:n_old].clone() if n_old else torch.zeros(0, 8)
        objects = {}
        for oid, po in s.last["per_obj"].items():
            row = rows[po["slot"]]
            objects[oid] = (row[:7].clone(), s.mask_bufs[po["slot"]][0]) if row[7] > 0 else (None, None)
        return dict(segmentation=s.seg, soft=s.soft[:len(self.obj_ids)], objects=objects, ids=self.obj_ids)

    def track_tensor(self, cur_frame, new_boxes_xyxy=None, init_mask=None):
        """cur_frame: preprocessed frame (fp32 NCHW or uint8 NHWC).  new_boxes_xyxy: dict obj_id -> box (resized-image coordinates)
        of objects that first appear in this frame, init_mask: their uint8 label map [H0,W0] (unicorn_vos.py:86-98).
        Returns dict(segmentation=uint8 [H0,W0] device tensor, soft=fp32 [n,H0,W0], objects={obj_id: (det_row [7] cpu | None,
        mask fp32 [H,W] device at network resolution | None)})."""
        assert self._ring.submitted == self._ring.collected, "collect() the frames in flight first"
        new_ids = list(new_boxes_xyxy.keys()) if new_boxes_xyxy else []
        if new_ids:
            assert init_mask is not None and init_mask.dtype == torch.uint8 and tuple(init_mask.shape) == self.orig_size
            init_mask = init_mask.to(self.eng.dev).contiguous()
        s = self._workers[0]
        self._enqueue(s, cur_frame, new_ids, new_boxes_xyxy, init_mask)
        return self._finish(s)

    # ------------------------------------------------------------------------------------------ frames in flight
    def submit(self, cur_frame):
        """Enqueue a steady-state frame (no new objects) in the next slot, on its stream; at most `depth` frames may be uncollected.
        The tensors of a collected result stay valid until that slot's next submit (`depth` submits later)."""
        s = self._ring.submit()
        if s.stream is not None:
            s.stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s.stream):
            self._enqueue(s, cur_frame)

    def collect(self):
        """Result of the oldest submitted frame (same dict as track_tensor)."""
        return self._finish(self._ring.collect())

    # ------------------------------------------------------------------------------------------ reference protocol
    def initialize(self, image, info: dict):
        """image: a raw frame, RGB uint8 [h, w, 3] or NV12 uint8 [3h/2, w] (letterbox_frame); info: init_object_ids, init_bbox {id:
        [x,y,w,h]} (unicorn_vos.py:43-69)."""
        ref, r, (self.H, self.W) = letterbox_frame(image, self.input_size, self.eng.dev)
        for oid in info["init_object_ids"]:
            self.state_pre_dict[oid] = info["init_bbox"][oid]
        boxes = {oid: xyxy_resized(info["init_bbox"][oid], r) for oid in info["init_object_ids"]}
        self.initialize_tensor(ref, boxes, orig_size=(self.H, self.W), r=r)

    def track(self, image, info: dict = None):
        """image: a raw frame as initialize() takes it -> {"segmentation": uint8 [H,W] numpy} (unicorn_vos.py:71-127)."""
        info = info or {}
        cur, r, _ = letterbox_frame(image, self.input_size, self.eng.dev)
        new_boxes, init_mask = None, None
        if "init_object_ids" in info:
            for oid in info["init_object_ids"]:
                self.state_pre_dict[oid] = info["init_bbox"][oid]
            new_boxes = {oid: xyxy_resized(info["init_bbox"][oid], r) for oid in info["init_object_ids"]}
            init_mask = torch.as_tensor(info["init_mask"]).to(torch.uint8)
        out = self.track_tensor(cur, new_boxes, init_mask)
        for oid, (det, _) in out["objects"].items():  # unicorn_vos.py:137-149 (state of the best instance, xywh ints)
            if det is not None:
                self.state_pre_dict[oid] = state_xywh(det, r, self.input_size)
        return {"segmentation": out["segmentation"].cpu().numpy()}


# ---------------------------------------------------------------------------------------------------------- several sequences
MAX_OBJECTS_PER_SEQUENCE = 16  # uc_vos_aggregate assembles at most 16 objects per frame
ROWS_PER_GROUP_SLOT = 8        # uc_corr_propagate carries at most 8 label rows per sequence


class _BatchSeq:
    """One sequence of UnicornVOSBatch: its reference groups in order (group slots, object ids) and the object slot of every id."""

    def __init__(self, orig_size, r):
        self.groups, self.obj_slot = [], {}
        self.orig_size, self.r = tuple(orig_size), float(r)
        self.seg = self.soft = None

    @property
    def obj_ids(self):
        return [o for _, ids in self.groups for o in ids]


class UnicornVOSBatch:
    """`n_seq` VOS sequences in lock step: one batched frame per step, captured as one CUDA graph.  The backbone and the mask branch
    run on the n_seq frames; every reference group of every sequence is a group slot of one batched interaction -> upsample ->
    correlation; every object of every sequence is an object slot of one batched head -> NMS -> dynamic-mask pass.  The result assembly
    (uc_vos_aggregate) then runs once per sequence at that sequence's original frame size.  Each sequence's label maps, soft masks
    and detection rows equal those of its own UnicornVOSTrack, bit for bit.

    Capacity is fixed at construction: every step computes all `max_objects` object slots and all `max_groups` group slots, and an
    unused slot computes on stale buffers whose results are discarded.  A reference group takes one group slot per 8 objects.  Which
    sequence, group slot and label row an object slot reads is device data (int32 tensors written in place), so initialising a
    sequence or adding objects writes into the static buffers the graph reads and never re-captures it.  A request beyond
    max_objects, max_groups or 16 objects in one sequence raises ValueError before any state changes."""

    def __init__(self, engine: UnicornEngine, input_size, n_seq, max_objects, max_groups, conf=0.001, nms=0.65, max_inst=1, d_rate=2,
                 use_graph=True):
        assert engine.cfg["mask"], "VOS needs a *_mask model"
        assert n_seq >= 1 and max_objects >= 1 and max_groups >= 1
        self.eng, self.input_size, self.n_seq = engine, tuple(input_size), n_seq
        self.max_objects, self.max_groups = max_objects, max_groups
        self.conf, self.nms, self.max_inst, self.d_rate = conf, nms, max_inst, d_rate
        self.use_graph = use_graph
        self.R = min(ROWS_PER_GROUP_SLOT, max_objects)  # label rows of every group slot (rows past a group's objects are ignored)
        H, W = self.input_size
        dev = engine.dev
        n8, n16 = (H // 8) * (W // 8), (H // 16) * (W // 16)
        self.slot = FrameSlot(engine, H, W, batch=n_seq)
        self._ref_slot = FrameSlot(engine, H, W)  # B = 1 reference frame of initialize_tensor
        self.ws = ops.PostWorkspace(anchor_count(H, W), dev, max_objects)
        self.ref_proj = tuple(torch.zeros(max_groups * n16, 256, dtype=torch.bfloat16, device=dev) for _ in range(2))
        self.lbs = torch.zeros(max_groups, self.R, n8, dtype=torch.float32, device=dev)
        i32 = dict(dtype=torch.int32, device=dev)
        self.group_seq = torch.zeros(max_groups, **i32)  # sequence whose frame each group slot reads
        self.obj_seq = torch.zeros(max_objects, **i32)  # sequence whose pyramid each object slot reads
        self.obj_row = torch.zeros(max_objects, **i32)  # group slot * R + label row of each object slot
        self.image_of = torch.full((max_objects,), -1, **i32)  # mask-branch image of each object slot, -1: unused (skipped)
        self.masks = torch.zeros(max_objects, 1, H, W, dtype=torch.float32, device=dev)
        self.rows = torch.zeros(max_objects, 8, dtype=torch.float32, device=dev)  # best detection row + count of each object slot
        self.host_rows = torch.zeros(max_objects, 8).pin_memory()
        self._frames = LetterboxBatch(n_seq, self.input_size, dev)  # the letterboxed frames of track()
        self._gs = [None] * max_groups  # host mirrors of the slot tables: sequence of a group slot, (sequence, group slot, row)
        self._os = [None] * max_objects
        self.seqs = [None] * n_seq
        self.state_pre_dicts = [{} for _ in range(n_seq)]
        self.launches_per_frame = 0

    # -------------------------------------------------------------------------------- slots
    def _check_capacity(self, requests):
        """requests: (sequence, objects to add, replace the sequence's objects).  Raises ValueError when they do not fit together."""
        free_g, free_o = self._gs.count(None), self._os.count(None)
        need_g = need_o = 0
        for i, n_new, replace in requests:
            sq = self.seqs[i]
            have = 0 if (replace or sq is None) else len(sq.obj_ids)
            if have + n_new > MAX_OBJECTS_PER_SEQUENCE:
                raise ValueError(f"UnicornVOSBatch: sequence {i} would track {have + n_new} objects (at most {MAX_OBJECTS_PER_SEQUENCE})")
            if replace and sq is not None:
                free_g += sum(len(g) for g, _ in sq.groups)
                free_o += len(sq.obj_slot)
            need_g += -(-n_new // ROWS_PER_GROUP_SLOT)
            need_o += n_new
        if need_o > free_o:
            raise ValueError(f"UnicornVOSBatch: {need_o} new objects but {free_o} of max_objects = {self.max_objects} slots are free")
        if need_g > free_g:
            raise ValueError(f"UnicornVOSBatch: {need_g} new group slots but {free_g} of max_groups = {self.max_groups} are free")

    def _release(self, i):
        self._gs = [None if s == i else s for s in self._gs]
        self._os = [None if o is not None and o[0] == i else o for o in self._os]
        self.seqs[i] = None

    def _add_group(self, i, ref_feat, boxes_xyxy):
        """Objects `boxes_xyxy` of sequence i with reference feature ref_feat [1,h,w,C]: project the reference once (B = 1), write it and
        the label values into free group slots (8 objects per slot) and give every object a free object slot."""
        e, sq = self.eng, self.seqs[i]
        ids = list(boxes_xyxy.keys())
        n16 = self.ref_proj[0].shape[0] // self.max_groups
        src, q = e.project_ref(ref_feat)
        lbs = label_values([boxes_xyxy[o] for o in ids], self.input_size, e.dev)
        gslots = []
        for c0 in range(0, len(ids), ROWS_PER_GROUP_SLOT):
            g = self._gs.index(None)
            self._gs[g] = i
            self.ref_proj[0][g * n16:(g + 1) * n16].copy_(src)
            self.ref_proj[1][g * n16:(g + 1) * n16].copy_(q)
            chunk = ids[c0:c0 + ROWS_PER_GROUP_SLOT]
            self.lbs[g].zero_()
            self.lbs[g, :len(chunk)].copy_(lbs[c0:c0 + len(chunk)])
            for row, oid in enumerate(chunk):
                o = self._os.index(None)
                self._os[o] = (i, g, row)
                sq.obj_slot[oid] = o
            gslots.append(g)
        sq.groups.append((gslots, ids))

    def _write_tables(self):
        """The slot tables the graph reads, from their host mirrors (in place: the captured graph stays valid)."""
        t = lambda v: torch.tensor(v, dtype=torch.int32)  # noqa: E731
        self.group_seq.copy_(t([0 if s is None else s for s in self._gs]))
        self.obj_seq.copy_(t([0 if o is None else o[0] for o in self._os]))
        self.obj_row.copy_(t([0 if o is None else o[1] * self.R + o[2] for o in self._os]))
        self.image_of.copy_(t([-1 if o is None else o[0] for o in self._os]))

    # -------------------------------------------------------------------------------- device-side frame
    def _frame(self):
        e = self.eng
        H, W = self.input_size
        hh, ww = H // 8, W // 8
        G, O, R = self.max_groups, self.max_objects, self.R
        F32 = torch.float32
        e.begin_frame()
        fpn, seq = e.backbone(self.slot.img, tag="cur")
        mf, um = e.mask_branch(fpn)  # once per sequence, shared by its objects through image_of
        feat = seq["feat"]
        feat_g = torch.index_select(feat, 0, self.group_seq, out=e.buf("vosb.feat", (G,) + tuple(feat.shape[1:]), feat.dtype))
        f_pre, f_cur = e.interaction(None, feat_g, ref_proj=self.ref_proj)
        e_pre, e_cur = e.upsample(f_pre, "embp"), e.upsample(f_cur, "embc")
        coarse = ops.corr_propagate(e_pre.view(G, -1, 128), e_cur.view(G, -1, 128), self.lbs, out=e.buf("vosb.coarse", (G, R, hh * ww), F32))
        c0 = torch.index_select(coarse.view(G * R, hh * ww), 0, self.obj_row, out=e.buf("vosb.c0", (O, hh * ww), F32)).view(O, hh, ww)
        pri = (c0, ops.bilinear(c0, hh // 2, ww // 2, 2.0, 2.0, out=e.buf("vosb.p1", (O, hh // 2, ww // 2), F32)),
               ops.bilinear(c0, hh // 4, ww // 4, 4.0, 4.0, out=e.buf("vosb.p2", (O, hh // 4, ww // 4), F32)))
        fpn_o = [torch.index_select(f, 0, self.obj_seq, out=e.buf(f"vosb.fpn{k}", (O,) + tuple(f.shape[1:]), f.dtype)) for k, f in enumerate(fpn)]
        head = e.head(fpn_o, pri, "sot", with_masks=True)
        ops.postprocess_device(head, 1, self.conf, self.nms, self.ws, max_keep=self.max_inst)
        self.masks.zero_()  # an object without a detection contributes an all-zero mask (unicorn_vos.py:154-155)
        up = 8 // self.d_rate
        hw = [(t.shape[1], t.shape[2]) for t in e.dyn_levels]
        ops.dynamic_masks(mf, um, e.dyn_levels, hw, self.ws, 1, up_rate=up, d_rate=self.d_rate, out=self.masks,
                          scratch=e.buf("vosb.scratch", (O * hh * ww * (1 + up * up),), F32), image_of=self.image_of)
        self.rows[:, :7].copy_(self.ws.dets.view(O, -1, 7)[:, 0])
        self.rows[:, 7].copy_(self.ws.count)
        self.slot.last = dict(feat=feat, mask_feats=mf, up_masks=um, coarse=coarse, head=head, dyn=list(e.dyn_levels))

    def _run(self):
        s = self.slot
        if not self.use_graph:
            self._frame()
        elif s.graph is None:
            s.graph, self.launches_per_frame = s.capture(self._frame, warmup=True)
        else:
            s.graph.replay()
        self.host_rows.copy_(self.rows, non_blocking=True)  # one read: every object slot's detection row and count
        torch.cuda.current_stream().synchronize()

    # -------------------------------------------------------------------------------- tensor protocol
    def initialize_tensor(self, i, ref_frame, boxes_xyxy, orig_size=None, r=1.0):
        """(Re)initialise sequence slot i: ref_frame preprocessed fp32 [1,3,H,W] or uint8 [1,H,W,3]; boxes_xyxy dict obj_id -> box in
        resized-image coordinates; orig_size = (height, width) of the original frames (default: the input size), r = letterbox ratio."""
        assert 0 <= i < self.n_seq and len(boxes_xyxy) >= 1
        self._check_capacity([(i, len(boxes_xyxy), True)])
        e = self.eng
        torch.cuda.synchronize()
        inp = self._ref_slot.stage(ref_frame)
        e.begin_frame()
        _, seq = e.backbone(inp, tag="ref")
        ref_feat = seq["feat"].clone()
        self._release(i)
        self.seqs[i] = _BatchSeq(orig_size if orig_size is not None else self.input_size, r)
        self._add_group(i, ref_feat, boxes_xyxy)
        self._write_tables()
        torch.cuda.synchronize()

    def track_tensor(self, frames, new=None):
        """frames: preprocessed [n_seq,H,W,3] uint8 / [n_seq,3,H,W] fp32, or a list of n_seq frames [1,...] with None for an idle slot.
        new: {slot: (boxes_xyxy, init_mask)} objects that first appear in that slot's frame (dict obj_id -> box in resized-image
        coordinates, uint8 label map [H0,W0]).  Returns n_seq results shaped like UnicornVOSTrack.track_tensor's, None for idle or
        uninitialised slots.  The returned device tensors are overwritten by the next step."""
        new = dict(new or {})
        n = self.n_seq
        if torch.is_tensor(frames):
            assert frames.shape[0] == n
            active = [True] * n
        else:
            assert len(frames) == n
            active = [f is not None for f in frames]
        for i in new:
            assert self.seqs[i] is not None and active[i], f"UnicornVOSBatch: new objects for slot {i}, which has no frame in this step"
        self._check_capacity([(i, len(b), False) for i, (b, _) in new.items()])
        inits = {}
        for i, (_, m) in new.items():
            assert m is not None and m.dtype == torch.uint8 and tuple(m.shape) == self.seqs[i].orig_size
            inits[i] = m.to(self.eng.dev).contiguous()
        if not any(active):
            return [None] * n
        if torch.is_tensor(frames):
            self.slot.stage(frames)
        else:
            buf = self.slot.use_u8(next(f for f in frames if f is not None).dtype == torch.uint8)
            for i, f in enumerate(frames):
                if f is not None:
                    buf[i:i + 1].copy_(f, non_blocking=True)
        self._run()
        H, W = self.input_size
        feat = self.slot.last["feat"]
        res = [None] * n
        for i, sq in enumerate(self.seqs):
            if sq is None or not active[i]:
                continue
            old = sq.obj_ids
            new_ids = list(new[i][0].keys()) if i in new else []
            ids = old + new_ids
            H0, W0 = sq.orig_size
            if sq.seg is None or sq.soft.shape[0] < len(ids):
                sq.seg = torch.zeros(H0, W0, dtype=torch.uint8, device=self.eng.dev)
                sq.soft = torch.zeros(max(len(ids), 4), H0, W0, dtype=torch.float32, device=self.eng.dev)
            ops.vos_aggregate([self.masks[sq.obj_slot[o]] for o in old], inits.get(i), ids, H, W, sq.r, sq.soft, sq.seg)
            objects = {}
            for o in old:
                k = sq.obj_slot[o]
                row = self.host_rows[k]
                objects[o] = (row[:7].clone(), self.masks[k, 0]) if row[7] > 0 else (None, None)
            if new_ids:  # this frame becomes the reference of the new objects (unicorn_vos.py:87-88)
                self._add_group(i, feat[i:i + 1].clone(), new[i][0])
            res[i] = dict(segmentation=sq.seg, soft=sq.soft[:len(sq.obj_ids)], objects=objects, ids=sq.obj_ids)
        if new:
            self._write_tables()
        return res

    # -------------------------------------------------------------------------------- reference protocol
    def initialize(self, i, image, info: dict):
        """Slot i: image a raw frame, RGB uint8 [h, w, 3] or NV12 uint8 [3h/2, w] (letterbox_frame); info: init_object_ids, init_bbox
        {id: [x,y,w,h]} (unicorn_vos.py:43-69)."""
        ref, r, size = letterbox_frame(image, self.input_size, self.eng.dev)
        boxes = {oid: xyxy_resized(info["init_bbox"][oid], r) for oid in info["init_object_ids"]}
        self.initialize_tensor(i, ref, boxes, orig_size=size, r=r)
        self.state_pre_dicts[i] = {oid: info["init_bbox"][oid] for oid in info["init_object_ids"]}

    def track(self, images, infos=None):
        """images: n_seq raw frames as initialize() takes them (RGB and NV12 may be mixed), None for an idle slot; infos: n_seq dicts
        as UnicornVOSTrack.track takes (or None).  Returns n_seq results {"segmentation": uint8 [H,W] numpy}, None for idle or
        uninitialised slots."""
        n = self.n_seq
        assert len(images) == n
        infos = infos or [None] * n
        frames, ratios, _ = self._frames(images)
        new = {}
        for i, info in enumerate(infos):
            if info and "init_object_ids" in info and images[i] is not None and self.seqs[i] is not None:
                new[i] = ({oid: xyxy_resized(info["init_bbox"][oid], ratios[i]) for oid in info["init_object_ids"]},
                          torch.as_tensor(info["init_mask"]).to(torch.uint8))
        out = self.track_tensor([frames[i:i + 1] if im is not None else None for i, im in enumerate(images)], new)
        res = [None] * n
        for i, o in enumerate(out):
            if o is None:
                continue
            if i in new:
                for oid in infos[i]["init_object_ids"]:
                    self.state_pre_dicts[i][oid] = infos[i]["init_bbox"][oid]
            for oid, (det, _) in o["objects"].items():  # unicorn_vos.py:137-149 (state of the best instance, xywh ints)
                if det is not None:
                    self.state_pre_dicts[i][oid] = state_xywh(det, ratios[i], self.input_size)
            res[i] = {"segmentation": o["segmentation"].cpu().numpy()}
        return res

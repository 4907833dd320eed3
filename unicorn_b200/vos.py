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
from .frames import FrameSlot, Ring, in_flight
from .sot import get_label_map, preprocess, state_xywh, xyxy_resized


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
        H, W = self.input_size
        maps = [ops.bilinear(get_label_map(b, H, W, self.eng.dev), H // 8, W // 8, 8.0, 8.0).reshape(1, -1) for b in boxes_xyxy]
        return torch.cat(maps, 0).contiguous()

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
        """image: RGB uint8 HWC; info: init_object_ids, init_bbox {id: [x,y,w,h]} (unicorn_vos.py:43-69)."""
        self.H, self.W = image.shape[:2]
        ref, r = preprocess(image, self.input_size)
        for oid in info["init_object_ids"]:
            self.state_pre_dict[oid] = info["init_bbox"][oid]
        boxes = {oid: xyxy_resized(info["init_bbox"][oid], r) for oid in info["init_object_ids"]}
        self.initialize_tensor(ref, boxes, orig_size=(self.H, self.W), r=r)

    def track(self, image, info: dict = None):
        """-> {"segmentation": uint8 [H,W] numpy} (unicorn_vos.py:71-127)."""
        info = info or {}
        cur, r = preprocess(image, self.input_size)
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

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
`submit(frame)` / `collect()` keep `depth` steady-state frames in flight, each on its own stream and engine context (worker drivers
on UnicornEngine.fork() that share the reference groups); frames that add objects go through track_tensor() with the pipeline drained.
"""
import ctypes

import torch

from . import _lib, ops
from .engine import UnicornEngine
from .sot import get_label_map, preprocess


class _Group:
    """Objects sharing one reference frame (unicorn_vos.py: out_dict_pre / out_dict_pre_new[i])."""

    def __init__(self, ref_feat, ref_proj, obj_ids, lbs):
        self.ref_feat, self.ref_proj, self.obj_ids, self.lbs = ref_feat, ref_proj, list(obj_ids), lbs


class UnicornVOSTrack:
    def __init__(self, engine: UnicornEngine, input_size, conf=0.001, nms=0.65, max_inst=1, d_rate=2, use_graph=False, depth=1):
        assert engine.cfg["mask"], "VOS needs a *_mask model"
        assert depth >= 1
        self.eng, self.input_size = engine, tuple(input_size)
        self.conf, self.nms, self.max_inst, self.d_rate = conf, nms, max_inst, d_rate
        self.num_classes = 1
        H, W = self.input_size
        dev = engine.dev
        A = (H // 8) * (W // 8) + (H // 16) * (W // 16) + (H // 32) * (W // 32)
        self.ws = ops.PostWorkspace(A, dev)
        self.img_in = torch.empty(1, 3, H, W, dtype=torch.float32, device=dev)
        self.img_in_u8 = torch.empty(1, H, W, 3, dtype=torch.uint8, device=dev)
        self._u8 = False
        self.use_graph = use_graph
        self._graph, self._graph_key = None, None
        self._mask_bufs, self._det_bufs = [], []   # per object slot: fp32 [1,H,W] best-instance mask, fp32 [8] = det row + count
        self._seg = self._soft = None
        self.groups = []
        self.state_pre_dict = {}
        self.frame_id = 0
        self.launches_per_frame = 0
        self.debug = False  # tests: keep per-object copies of the head output and the controller maps
        self.last = {}
        self._rows_host, self._rows_ev, self._pending = None, torch.cuda.Event(), None
        # frames in flight: worker 0 is this driver, the others are drivers on engine forks sharing groups / geometry
        self.depth = depth
        self._stream = torch.cuda.Stream(device=dev) if depth > 1 else None
        self._workers = [self] + [UnicornVOSTrack(engine.fork(), input_size, conf, nms, max_inst, d_rate, use_graph, depth=1) for _ in range(depth - 1)]
        for w in self._workers[1:]:
            w._stream = torch.cuda.Stream(device=dev)
        self._submitted = self._collected = 0

    # ------------------------------------------------------------------------------------------ helpers
    def _stage_input(self, frame):
        u8 = frame.dtype == torch.uint8
        if u8 != self._u8:
            self._u8, self._graph = u8, None
        buf = self.img_in_u8 if u8 else self.img_in
        buf.copy_(frame, non_blocking=True)
        return buf

    def _label_maps(self, boxes_xyxy):
        H, W = self.input_size
        maps = [ops.bilinear(get_label_map(b, H, W, self.eng.dev), H // 8, W // 8, 8.0, 8.0).reshape(1, -1) for b in boxes_xyxy]
        return torch.cat(maps, 0).contiguous()

    def _slot(self, i):
        H, W = self.input_size
        while len(self._mask_bufs) <= i:
            self._mask_bufs.append(torch.zeros(1, H, W, dtype=torch.float32, device=self.eng.dev))
            self._det_bufs.append(torch.zeros(8, dtype=torch.float32, device=self.eng.dev))
        return self._mask_bufs[i], self._det_bufs[i]

    @property
    def obj_ids(self):
        return [o for g in self.groups for o in g.obj_ids]

    # ------------------------------------------------------------------------------------------ tensor protocol
    def initialize_tensor(self, ref_frame, boxes_xyxy, orig_size=None, r=1.0):
        """ref_frame: preprocessed fp32 [1,3,H,W] or uint8 [1,H,W,3]; boxes_xyxy: dict obj_id -> box in resized-image coordinates
        (unicorn_vos.py:60-66); orig_size = (height, width) of the original frames (default: the network input size), r = resize
        ratio of the letterbox."""
        e = self.eng
        inp = self._stage_input(ref_frame)
        e.begin_frame()
        _, seq = e.backbone(inp, tag="ref")
        ids = list(boxes_xyxy.keys())
        ref_feat = seq["feat"].clone()
        self.groups = [_Group(ref_feat, e.project_ref(ref_feat), ids, self._label_maps([boxes_xyxy[o] for o in ids]))]
        self.orig_size = tuple(orig_size) if orig_size is not None else self.input_size
        self.r = float(r)
        for w in self._workers:
            w._graph, w.frame_id, w._pending = None, 0, None
        self._submitted = self._collected = 0
        torch.cuda.synchronize()

    def _device_frame(self):
        """Every kernel of one steady-state frame (no host synchronisation; CUDA-graph capturable)."""
        e = self.eng
        H, W = self.input_size
        hh, ww = H // 8, W // 8
        e.begin_frame()
        fpn, seq = e.backbone(self.img_in_u8 if self._u8 else self.img_in, tag="cur")
        mf, um = e.mask_branch(fpn)  # identical for every object: computed once per frame
        self.last = dict(mask_feats=mf, up_masks=um, per_obj={}, feat=seq["feat"], coarse={})
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
                    ops.postprocess_device(head[0], 1, self.conf, self.nms, self.ws, max_keep=self.max_inst)
                    mask, det = self._slot(slot)
                    mask.zero_()  # an object without a detection contributes an all-zero mask (unicorn_vos.py:154-155)
                    hw = [(t.shape[1], t.shape[2]) for t in e.dyn_levels]
                    up = 8 // self.d_rate
                    ops.dynamic_masks(mf, um, e.dyn_levels, hw, self.ws, 1, up_rate=up, d_rate=self.d_rate, out=mask,
                                      scratch=e.buf("vos.scratch", (hh * ww * (1 + up * up),), torch.float32))
                    det[:7].copy_(self.ws.dets[0])
                    det[7:8].copy_(self.ws.count.view(1).float())
                    keep = (lambda t: t.clone()) if self.debug else (lambda t: t)
                    self.last["per_obj"][oid] = dict(head=keep(head), dyn=[keep(t) for t in e.dyn_levels], slot=slot)
                    self.last["coarse"][oid] = c
                    slot += 1
        return seq

    def _aggregate(self, new_ids=(), init_mask=None):
        """unicorn_vos.py:100-127 on the device.  Returns (segmentation uint8 [H0,W0], soft masks fp32 [n,H0,W0])."""
        H, W = self.input_size
        H0, W0 = self.orig_size
        ids = self.obj_ids + list(new_ids)
        n = len(ids)
        if self._seg is None or self._seg.shape != (H0, W0) or self._soft.shape[0] < n:
            self._seg = torch.zeros(H0, W0, dtype=torch.uint8, device=self.eng.dev)
            self._soft = torch.zeros(max(n, 4), H0, W0, dtype=torch.float32, device=self.eng.dev)
        objs = (_lib.UcVosObject * n)()
        n_old = len(self.obj_ids)
        for k, oid in enumerate(ids):
            objs[k].id = int(oid)
            if k < n_old:
                objs[k].mask = self._mask_bufs[k].data_ptr()
            else:
                objs[k].init_mask = init_mask.data_ptr()
        _lib.check(_lib.lib().uc_vos_aggregate(objs, n, H, W, H0, W0, ctypes.c_float(self.r), ctypes.c_void_p(self._soft.data_ptr()),
                                               ctypes.c_void_p(self._seg.data_ptr()), _lib.stream_ptr()), "uc_vos_aggregate")
        return self._seg, self._soft[:n]

    def _enqueue(self, cur_frame, new_ids=(), new_boxes_xyxy=None, init_mask=None):
        """Device half of a frame on the current stream + the asynchronous read of the detection rows; no host synchronisation
        unless a graph has to be (re)captured."""
        e = self.eng
        self.frame_id += 1
        self._stage_input(cur_frame)
        key = tuple(len(g.obj_ids) for g in self.groups)
        if self.use_graph and not new_ids and self.frame_id > 1:
            if self._graph is None or self._graph_key != key:
                self._device_frame()  # warm-up: buffers, kernel attributes, plan-time autotuning
                self._aggregate()
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                l0 = _lib.LAUNCHES
                with (torch.cuda.graph(g) if self._stream is None else torch.cuda.graph(g, stream=self._stream)):
                    self._device_frame()
                    self._aggregate()
                self.launches_per_frame = _lib.LAUNCHES - l0
                self._graph, self._graph_key, self._graph_last = g, key, self.last
            self._graph.replay()
            self.last = self._graph_last
            seg, soft = self._seg, self._soft[:len(self.obj_ids)]
        else:
            seq = self._device_frame()
            seg, soft = self._aggregate(new_ids, init_mask)
            if new_ids:  # this frame becomes the reference of the new objects (unicorn_vos.py:87-88)
                ref_feat = seq["feat"].clone()
                self.groups.append(_Group(ref_feat, e.project_ref(ref_feat), new_ids, self._label_maps([new_boxes_xyxy[o] for o in new_ids])))
                self._graph = None
        n_old = len(self.last["per_obj"])
        if n_old:  # one D2H read: detection rows + counts, into pinned memory
            if self._rows_host is None or self._rows_host.shape[0] < n_old:
                self._rows_host = torch.zeros(max(n_old, 4), 8).pin_memory()
            self._rows_host[:n_old].copy_(torch.stack(self._det_bufs[:n_old]), non_blocking=True)
        self._rows_ev.record()
        self._pending = (seg, soft, n_old, bool(new_ids))

    def _finish(self):
        seg, soft, n_old, had_new = self._pending
        self._pending = None
        self._rows_ev.synchronize()
        rows = self._rows_host[:n_old].clone() if n_old else torch.zeros(0, 8)
        objects = {}
        for oid, po in self.last["per_obj"].items():
            row = rows[po["slot"]]
            objects[oid] = (row[:7].clone(), self._mask_bufs[po["slot"]][0]) if row[7] > 0 else (None, None)
        return dict(segmentation=seg, soft=soft, objects=objects, ids=self.obj_ids)

    def track_tensor(self, cur_frame, new_boxes_xyxy=None, init_mask=None):
        """cur_frame: preprocessed frame (fp32 NCHW or uint8 NHWC).  new_boxes_xyxy: dict obj_id -> box (resized-image coordinates)
        of objects that first appear in this frame, init_mask: their uint8 label map [H0,W0] (unicorn_vos.py:86-98).
        Returns dict(segmentation=uint8 [H0,W0] device tensor, soft=fp32 [n,H0,W0], objects={obj_id: (det_row [7] cpu | None,
        mask fp32 [H,W] device at network resolution | None)})."""
        assert self._submitted == self._collected, "collect() the frames in flight first"
        new_ids = list(new_boxes_xyxy.keys()) if new_boxes_xyxy else []
        if new_ids:
            assert init_mask is not None and init_mask.dtype == torch.uint8 and tuple(init_mask.shape) == self.orig_size
            init_mask = init_mask.to(self.eng.dev).contiguous()
        self._enqueue(cur_frame, new_ids, new_boxes_xyxy, init_mask)
        return self._finish()

    # ------------------------------------------------------------------------------------------ frames in flight
    def submit(self, cur_frame):
        """Enqueue a steady-state frame (no new objects) on the next worker's stream; at most `depth` frames may be uncollected.
        The tensors of a collected result stay valid until that worker's next submit (`depth` submits later)."""
        assert self._submitted - self._collected < self.depth, "collect() a frame first"
        w = self._workers[self._submitted % self.depth]
        self._submitted += 1
        if w is not self:  # shared reference state and geometry
            w.groups, w.orig_size, w.r = self.groups, self.orig_size, self.r
        if w._stream is None:
            return w._enqueue(cur_frame)
        w._stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(w._stream):
            w._enqueue(cur_frame)

    def collect(self):
        """Result of the oldest submitted frame (same dict as track_tensor)."""
        assert self._collected < self._submitted, "nothing submitted"
        w = self._workers[self._collected % self.depth]
        self._collected += 1
        return w._finish()

    # ------------------------------------------------------------------------------------------ reference protocol
    def initialize(self, image, info: dict):
        """image: RGB uint8 HWC; info: init_object_ids, init_bbox {id: [x,y,w,h]} (unicorn_vos.py:43-69)."""
        self.H, self.W = image.shape[:2]
        ref, r = preprocess(image, self.input_size)
        boxes = {}
        for oid in info["init_object_ids"]:
            self.state_pre_dict[oid] = info["init_bbox"][oid]
            b = torch.tensor(info["init_bbox"][oid], dtype=torch.float32).view(-1)
            b[2:] += b[:2]
            boxes[oid] = b * r
        self.initialize_tensor(ref, boxes, orig_size=(self.H, self.W), r=r)

    def track(self, image, info: dict = None):
        """-> {"segmentation": uint8 [H,W] numpy} (unicorn_vos.py:71-127)."""
        info = info or {}
        cur, r = preprocess(image, self.input_size)
        new_boxes, init_mask = None, None
        if "init_object_ids" in info:
            new_boxes = {}
            for oid in info["init_object_ids"]:
                self.state_pre_dict[oid] = info["init_bbox"][oid]
                b = torch.tensor(info["init_bbox"][oid], dtype=torch.float32).view(-1)
                b[2:] += b[:2]
                new_boxes[oid] = b * r
            init_mask = torch.as_tensor(info["init_mask"]).to(torch.uint8)
        out = self.track_tensor(cur, new_boxes, init_mask)
        H, W = self.input_size
        for oid, (det, _) in out["objects"].items():  # unicorn_vos.py:137-149 (state of the best instance, xywh ints)
            if det is not None:
                b = det[:4].clone()
                b[0::2] = b[0::2].clamp(0, W)
                b[1::2] = b[1::2].clamp(0, H)
                b = (b / r).numpy()
                self.state_pre_dict[oid] = [int(b[0]), int(b[1]), int(b[2] - b[0]), int(b[3] - b[1])]
        return {"segmentation": out["segmentation"].cpu().numpy()}

"""SOT per-frame driver on the H100 engine — mirrors external/lib/test/tracker/unicorn_sot.py
(UnicornSOTTrack.initialize :39-56, track :57-77, get_det_results :78-109, PreprocessorX :111-123,
get_label_map :128-139) with the same initialize/track protocol (external/lib/test/tracker/basetracker.py:14-20).

What changes relative to the reference loop: the reference frame's projection is cached, the whole steady-state
frame (backbone -> interaction -> 2x upsample -> fused correlation -> head -> NMS) is one CUDA graph replay, and the
only per-frame host traffic is the input frame (pinned H2D) and the top-`max_inst` detection rows (D2H)."""
import torch

from . import ops
from .engine import UnicornEngine
from .frames import FrameSlot, Ring, in_flight


def get_label_map(box_xyxy, H, W, device):
    """unicorn_sot.py:128-139."""
    labels = torch.zeros((1, 1, H, W), dtype=torch.float32, device=device)
    x1, y1, x2, y2 = torch.round(torch.as_tensor(box_xyxy, dtype=torch.float32)).int().tolist()
    x1, x2 = max(0, min(x1, W)), max(0, min(x2, W))
    y1, y2 = max(0, min(y1, H)), max(0, min(y2, H))
    labels[0, 0, y1:y2, x1:x2] = 1.0
    return labels


def preprocess(img_rgb, input_size, out=None):
    """PreprocessorX.process (unicorn_sot.py:114-123): RGB uint8 HWC -> BGR letterboxed (pad 114), kept as uint8 HWC
    [1,H,W,3] (the float conversion and the HWC->CHW permute happen inside the stem kernel; values are identical to the
    reference's float tensor because cv2.resize already returns uint8).  Returns (tensor, r)."""
    import cv2
    height, width = img_rgb.shape[:2]
    r = min(input_size[0] / height, input_size[1] / width)
    rsz = cv2.resize(cv2.cvtColor(img_rgb, cv2.COLOR_RGB2BGR), (int(width * r), int(height * r)), interpolation=cv2.INTER_LINEAR)
    if out is None:
        out = torch.empty(1, input_size[0], input_size[1], 3, dtype=torch.uint8).pin_memory()
    out.fill_(114)
    out[0, :int(height * r), :int(width * r)] = torch.from_numpy(rsz)
    return out, r


def xyxy_resized(xywh, r):
    """Reference-protocol box [x, y, w, h] in original-image pixels -> [x1, y1, x2, y2] in resized-image coordinates
    (unicorn_sot.py:44-46, unicorn_vos.py:62-64)."""
    b = torch.tensor(xywh, dtype=torch.float32).view(-1)
    b[2:] += b[:2]
    return b * r


def state_xywh(det, r, input_size):
    """Detection row (corners in resized-image coordinates) -> the reference's state: corners clipped to the input, scaled back to
    the original image, [x, y, w, h] as ints (unicorn_sot.py:64-75, unicorn_vos.py:132-143)."""
    H, W = input_size
    b = det[:4].clone()
    b[0::2] = b[0::2].clamp(0, W)
    b[1::2] = b[1::2].clamp(0, H)
    b = (b / r).numpy()
    return [int(b[0]), int(b[1]), int(b[2] - b[0]), int(b[3] - b[1])]


class _Ctx(FrameSlot):
    """A frame slot plus the pinned read-back of its detection count and top `max_inst` rows."""

    def __init__(self, eng, H, W, stream, max_inst):
        super().__init__(eng, H, W, stream)
        self.host_dets = torch.empty(max_inst, 7, dtype=torch.float32).pin_memory()
        self.host_count = torch.zeros(1, dtype=torch.int32).pin_memory()


class UnicornSOTTrack:
    def __init__(self, engine: UnicornEngine, input_size, conf=0.001, nms=0.65, max_inst=3, use_graph=True, full_nms=False,
                 device_preproc=False, depth=1):
        """depth > 1: that many frames may be in flight (submit / collect), each on its own stream and engine context.  The frames
        of a sequence are independent — the network never sees the previous frame's result (unicorn_sot.py:57-109 uses only the
        initial frame's features and label map) — so overlapping them changes no output, only fills the SMs that one frame's
        small kernels and launch gaps leave idle.  track() / track_tensor() stay synchronous (one frame in, its result out)."""
        self.eng, self.input_size = engine, tuple(input_size)
        self.confthre, self.nmsthre, self.max_inst = conf, nms, max_inst
        self.num_classes = 1
        self.use_graph = use_graph
        # device_preproc: initialize()/track() upload the raw RGB frame and letterbox it on the GPU (uc_letterbox_u8, bit-exact
        # restatement of the reference's cv2 recipe) instead of resizing on the host
        self.device_preproc = device_preproc
        self._raw = None
        # the driver consumes output[:max_inst] only (unicorn_sot.py:69-70): stop the greedy NMS scan there.
        # full_nms=True reproduces the complete postprocess() list (used by the parity tests).
        self.nms_keep = 0 if full_nms else max_inst
        H, W = self.input_size
        assert depth >= 1
        self.depth = depth
        self._ring = Ring(in_flight(engine, depth, lambda eng, stream: _Ctx(eng, H, W, stream, max_inst)))
        self._ctxs = self._ring.slots  # bench.py reads pipe._ctxs[i]
        self.state = None
        self.frame_id = 0
        self.launches_per_frame = 0  # bench.py reads it

    # attributes of the single-context tracker (tests / bench read them): context 0
    img_in = property(lambda self: self._ctxs[0].img_in)
    img_in_u8 = property(lambda self: self._ctxs[0].img_in_u8)
    ws = property(lambda self: self._ctxs[0].ws)
    host_dets = property(lambda self: self._ctxs[0].host_dets)
    host_count = property(lambda self: self._ctxs[0].host_count)
    graph = property(lambda self: self._ctxs[0].graph)
    last = property(lambda self: self._ctxs[(max(self._ring.collected, 1) - 1) % self.depth].last)

    # -------------------------------------------------------------------------------- device-side frame
    def _frame(self, c):
        e = c.eng
        e.begin_frame()
        def correlate(seq):  # runs on a second stream while the neck runs on the main one
            f_pre, f_cur = e.interaction(self.ref_feat, seq["feat"], ref_proj=self.ref_proj)
            e_pre, e_cur = e.upsample(f_pre, "embp"), e.upsample(f_cur, "embc")
            return f_pre, f_cur, e_pre, e_cur, e.propagate(e_pre, e_cur, self.lbs_pre)

        fpn, seq, (f_pre, f_cur, e_pre, e_cur, priors) = e.backbone(c.img, tag="cur", side=correlate)
        out = e.head(fpn, priors, "sot")
        ops.postprocess_device(out[0], 1, self.confthre, self.nmsthre, c.ws, max_keep=self.nms_keep)
        c.last = dict(fpn=fpn, feat=seq["feat"], inter_pre=f_pre, inter_cur=f_cur, embed_pre=e_pre, embed_cur=e_cur, priors=priors, head=out)

    def initialize_tensor(self, ref_frame, init_box_xyxy):
        """ref_frame: preprocessed fp32 [1,3,H,W] or uint8 [1,H,W,3] (host or device); init box in resized-image coordinates."""
        e = self.eng
        H, W = self.input_size
        torch.cuda.synchronize()
        inp = self._ctxs[0].stage(ref_frame)
        e.begin_frame()
        _, seq = e.backbone(inp, tag="ref")
        self.ref_feat = seq["feat"].clone()
        self.ref_proj = e.project_ref(self.ref_feat)  # this tracker's own copy (several trackers may share the engine)
        lab = get_label_map(init_box_xyxy, H, W, e.dev)
        self.lbs_pre = ops.bilinear(lab, H // 8, W // 8, 8.0, 8.0).reshape(1, -1).contiguous()
        self._ring.reset()
        self.frame_id = 0
        torch.cuda.synchronize()

    def track_tensor(self, cur_frame):
        """cur_frame: preprocessed fp32 [1,3,H,W] or uint8 [1,H,W,3], ideally pinned host memory.  Returns (dets[:max_inst] cpu, count)."""
        self.submit(cur_frame)
        return self.collect()

    def submit(self, cur_frame):
        """Pipelined protocol: enqueue a frame (returns immediately); at most `depth` frames may be uncollected.  On the context's
        stream: input copy, graph replay (or eager launches), asynchronous read-back of (count, top rows) into the context's pinned
        slot.  A context's first graph frame is warm-up, capture and replay in one call, so the graph exists after one frame."""
        c = self._ring.submit()
        self.frame_id = self._ring.submitted
        with torch.cuda.stream(c.stream):  # None: the current stream
            c.stage(cur_frame)
            if not self.use_graph:
                self._frame(c)
            elif c.graph is None:
                c.graph, self.launches_per_frame = c.capture(lambda: self._frame(c), warmup=True)
            else:
                c.graph.replay()
            c.host_count.copy_(c.ws.count, non_blocking=True)
            c.host_dets.copy_(c.ws.dets[:self.max_inst], non_blocking=True)
            c.event.record()

    def collect(self):
        """Result of the oldest submitted frame: (dets[:max_inst] cpu, count)."""
        c = self._ring.collect()
        c.event.synchronize()
        n = int(c.host_count.item())
        return c.host_dets[:min(n, self.max_inst)].clone(), n

    # -------------------------------------------------------------------------------- reference protocol
    def _preprocess(self, image):
        if not self.device_preproc:
            return preprocess(image, self.input_size)
        src = torch.from_numpy(image) if not torch.is_tensor(image) else image
        assert src.dtype == torch.uint8 and src.dim() == 3 and src.shape[2] == 3
        if self._raw is None or self._raw.shape != src.shape:
            self._raw = torch.empty(src.shape, dtype=torch.uint8, device=self.eng.dev)
            self._raw_host = torch.empty(src.shape, dtype=torch.uint8).pin_memory()
        self._raw_host.copy_(src)
        self._raw.copy_(self._raw_host, non_blocking=True)
        return ops.letterbox_u8(self._raw, self.input_size, swap_rb=True)  # uint8 [1,H,W,3] on the device

    def initialize(self, image, info: dict):
        ref, r = self._preprocess(image)
        self.initialize_tensor(ref, xyxy_resized(info["init_bbox"], r))
        self.state = info["init_bbox"]

    def track(self, image, info: dict = None):
        cur, r = self._preprocess(image)
        dets, n = self.track_tensor(cur)
        if n > 0:
            self.state = state_xywh(dets[0], r, self.input_size)
        return {"target_bbox": self.state}


class UnicornSOTBatch:
    """`n_seq` SOT sequences in lock step: one batched frame (backbone -> interaction -> upsample -> correlation -> head -> NMS over
    all sequences) per step, captured as one CUDA graph.  Each sequence's results equal those of its own UnicornSOTTrack: every
    kernel of the batched frame computes each image as its B = 1 launch does.

    initialize(i, ...) sets sequence slot i at any time: its reference frame runs at B = 1 and its reference projection and label
    values are written in place into the static batched buffers the graph reads, so the graph stays valid and the other slots are
    unaffected.  A slot that has not been initialised, or gets None in track(), computes on whatever its input buffer holds and its
    result is discarded."""

    def __init__(self, engine: UnicornEngine, input_size, n_seq, conf=0.001, nms=0.65, max_inst=3, use_graph=True, device_preproc=False):
        assert n_seq >= 1
        self.eng, self.input_size, self.n_seq = engine, tuple(input_size), n_seq
        self.confthre, self.nmsthre, self.max_inst = conf, nms, max_inst
        self.use_graph, self.device_preproc = use_graph, device_preproc
        H, W = self.input_size
        dev = engine.dev
        self.slot = FrameSlot(engine, H, W, batch=n_seq)
        self._ref_slot = FrameSlot(engine, H, W)  # B = 1 input of initialize
        n16 = (H // 16) * (W // 16)
        self.ref_proj = (torch.zeros(n_seq * n16, 256, dtype=torch.bfloat16, device=dev), torch.zeros(n_seq * n16, 256, dtype=torch.bfloat16, device=dev))
        self.lbs_pre = torch.zeros(n_seq, 1, (H // 8) * (W // 8), dtype=torch.float32, device=dev)
        self.host_dets = torch.empty(n_seq, max_inst, 7, dtype=torch.float32).pin_memory()
        self.host_count = torch.zeros(n_seq, dtype=torch.int32).pin_memory()
        self._host_in = torch.full((n_seq, H, W, 3), 114, dtype=torch.uint8).pin_memory()  # host-letterboxed frames (track())
        self._raw = [None] * n_seq
        self.ready = [False] * n_seq
        self.states = [None] * n_seq
        self.launches_per_frame = 0

    # -------------------------------------------------------------------------------- device-side frame
    def _frame(self):
        e, n = self.eng, self.n_seq
        e.begin_frame()
        values = self.lbs_pre if n > 1 else self.lbs_pre[0]

        def correlate(seq):
            f_pre, f_cur = e.interaction(None, seq["feat"], ref_proj=self.ref_proj)
            e_pre, e_cur = e.upsample(f_pre, "embp"), e.upsample(f_cur, "embc")
            return e.propagate(e_pre, e_cur, values)

        fpn, seq, priors = e.backbone(self.slot.img, tag="cur", side=correlate)
        out = e.head(fpn, priors, "sot")
        ops.postprocess_device(out, 1, self.confthre, self.nmsthre, self.slot.ws, max_keep=self.max_inst)
        self.slot.last = dict(fpn=fpn, feat=seq["feat"], priors=priors, head=out)

    def _run(self):
        s = self.slot
        if not self.use_graph:
            self._frame()
        elif s.graph is None:
            s.graph, self.launches_per_frame = s.capture(self._frame, warmup=True)
        else:
            s.graph.replay()
        dets = s.ws.dets.view(self.n_seq, -1, 7)
        self.host_count.copy_(s.ws.count, non_blocking=True)
        self.host_dets.copy_(dets[:, :self.max_inst], non_blocking=True)
        torch.cuda.current_stream().synchronize()

    def initialize_tensor(self, i, ref_frame, init_box_xyxy):
        """Slot i: ref_frame preprocessed fp32 [1,3,H,W] or uint8 [1,H,W,3] (host or device); init box in resized-image coordinates."""
        assert 0 <= i < self.n_seq
        e = self.eng
        H, W = self.input_size
        n16 = (H // 16) * (W // 16)
        torch.cuda.synchronize()
        inp = self._ref_slot.stage(ref_frame)
        e.begin_frame()
        _, seq = e.backbone(inp, tag="ref")
        src, q = e.project_ref(seq["feat"])
        self.ref_proj[0][i * n16:(i + 1) * n16].copy_(src)
        self.ref_proj[1][i * n16:(i + 1) * n16].copy_(q)
        lab = get_label_map(init_box_xyxy, H, W, e.dev)
        self.lbs_pre[i].copy_(ops.bilinear(lab, H // 8, W // 8, 8.0, 8.0).reshape(1, -1))
        self.ready[i] = True
        torch.cuda.synchronize()

    def track_tensor(self, frames):
        """frames: [n_seq,H,W,3] uint8 or [n_seq,3,H,W] fp32 preprocessed (ideally pinned host memory).  Returns (dets
        [n_seq, max_inst, 7], counts [n_seq]) on the host; rows past a sequence's count are stale."""
        self.slot.stage(frames)
        self._run()
        return self.host_dets.clone(), self.host_count.clone()

    # -------------------------------------------------------------------------------- reference protocol
    def initialize(self, i, image, info: dict):
        if self.device_preproc:
            ref, r = self._device_letterbox(i, image, None)
        else:
            ref, r = preprocess(image, self.input_size)
        self.initialize_tensor(i, ref, xyxy_resized(info["init_bbox"], r))
        self.states[i] = info["init_bbox"]

    def _device_letterbox(self, i, image, out):
        src = torch.from_numpy(image) if not torch.is_tensor(image) else image
        assert src.dtype == torch.uint8 and src.dim() == 3 and src.shape[2] == 3
        if self._raw[i] is None or self._raw[i][0].shape != src.shape:
            self._raw[i] = (torch.empty(src.shape, dtype=torch.uint8, device=self.eng.dev), torch.empty(src.shape, dtype=torch.uint8).pin_memory())
        dev_raw, host_raw = self._raw[i]
        host_raw.copy_(src)
        dev_raw.copy_(host_raw, non_blocking=True)
        return ops.letterbox_u8(dev_raw, self.input_size, swap_rb=True, out=out)

    def track(self, images):
        """images: n_seq RGB frames (HWC uint8), None for an idle slot.  Returns n_seq results {"target_bbox": [x, y, w, h]}, None for
        idle or uninitialised slots."""
        assert len(images) == self.n_seq
        ratios = [None] * self.n_seq
        if self.device_preproc:
            buf = self.slot.use_u8(True)
            for i, im in enumerate(images):
                if im is not None:
                    ratios[i] = self._device_letterbox(i, im, buf[i:i + 1])[1]
            self._run()
        else:
            for i, im in enumerate(images):
                if im is not None:
                    ratios[i] = preprocess(im, self.input_size, out=self._host_in[i:i + 1])[1]
            self.slot.stage(self._host_in)
            self._run()
        res = [None] * self.n_seq
        for i, r in enumerate(ratios):
            if r is None or not self.ready[i]:
                continue
            n = int(self.host_count[i])
            if n > 0:
                self.states[i] = state_xywh(self.host_dets[i, 0], r, self.input_size)
            res[i] = {"target_bbox": self.states[i]}
        return res

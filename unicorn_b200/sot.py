"""SOT per-frame driver on the H100 engine — mirrors external/lib/test/tracker/unicorn_sot.py
(UnicornSOTTrack.initialize :39-56, track :57-77, get_det_results :78-109, PreprocessorX :111-123,
get_label_map :128-139) with the same initialize/track protocol (external/lib/test/tracker/basetracker.py:14-20).

What changes relative to the reference loop: the reference frame's projection is cached, the whole steady-state
frame (backbone -> interaction -> 2x upsample -> fused correlation -> head -> NMS) is one CUDA graph replay, and the
only per-frame host traffic is the input frame (pinned H2D) and the top-`max_inst` detection rows (D2H).

UnicornSOTBatch is the driver: `n_seq` sequences in lock step, one batched frame per step, optionally several steps in flight.
UnicornSOTTrack is its n_seq = 1 case under the reference's one-sequence protocol."""
import torch

from . import ops, shared_ops
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


def nv12_size(image):
    """(h, w) of a 2-D frame, which is NV12: uint8 [3h/2, w] (numpy array or tensor), h rows of luma then h/2 rows of interleaved
    U, V, with h and w even.  None for a frame that is not 2-D (an RGB frame, checked by the path that reads it).  ValueError for
    any other 2-D frame."""
    if getattr(image, "ndim", None) != 2:
        return None
    rows, w = (int(v) for v in image.shape)
    h = rows * 2 // 3
    if str(image.dtype) not in ("uint8", "torch.uint8") or rows % 3 or h < 2 or h % 2 or w < 2 or w % 2:
        raise ValueError(f"a 2-D frame is NV12, uint8 [3h/2, w] with h and w even and >= 2; got {tuple(image.shape)} {image.dtype}")
    return h, w


def letterbox_frame(image, input_size, device, out=None, device_out=None, device_preproc=False, rgb=True):
    """One raw frame -> (letterboxed BGR uint8 [1,H,W,3], r, (h, w) of the original frame).  The one place that knows the frame
    formats the drivers take:
      * uint8 [h, w, 3], RGB as the reference's frames (rgb=False: BGR, as cv2 loads images): preprocess() with cv2 on the host into
        `out`, or with device_preproc uploaded and letterboxed on `device` (uc_letterbox_u8) into `device_out`;
      * uint8 [3h/2, w], NV12 as hardware decoders deliver frames: always letterboxed on `device` (uc_letterbox_nv12) into
        `device_out`, to the bytes the RGB frame cv2.cvtColor(image, COLOR_YUV2RGB_NV12) gives.  rgb does not apply.
    A CUDA tensor on `device` is read in place on the current stream, which it is recorded on, so its memory is not reused before
    that read even when the caller drops it right away; one on another GPU is copied over.  A host array or tensor is staged through
    pinned memory (1.5 bytes per pixel for NV12).  A destination left None is allocated.  A malformed 2-D frame raises ValueError
    before anything is enqueued."""
    size = nv12_size(image)
    if size is None and not device_preproc:
        assert rgb, "a BGR frame is letterboxed on the device"
        frame, r = preprocess(image, input_size, out=out)
        return frame, r, tuple(image.shape[:2])
    device = torch.device(device)
    if device.index is None:
        device = torch.device(device.type, torch.cuda.current_device())
    src = torch.as_tensor(image)
    if src.device == device:
        src.record_stream(torch.cuda.current_stream(device))
    else:
        if not src.is_cuda and not src.is_pinned():
            src = torch.empty(src.shape, dtype=src.dtype, pin_memory=True).copy_(src)
        src = src.to(device, non_blocking=True)
    if size is not None:
        frame, r = shared_ops.letterbox_nv12(src, input_size, out=device_out)
        return frame, r, size
    assert src.dtype == torch.uint8 and src.dim() == 3 and src.shape[2] == 3
    frame, r = ops.letterbox_u8(src.contiguous(), input_size, swap_rb=rgb, out=device_out)
    return frame, r, tuple(src.shape[:2])


class LetterboxBatch:
    """The raw frames of one batched step, letterboxed (letterbox_frame) into one uint8 [n,H,W,3] batch.  A frame letterboxed on the
    host lands in a pinned buffer, one letterboxed on the device in a device buffer, allocated by the first step that needs it.  The
    batch is the pinned buffer when no frame of the step was letterboxed on the device, otherwise the device buffer with the
    host-letterboxed frames copied up, so RGB and NV12 frames mix in one step."""

    def __init__(self, n, input_size, device, device_preproc=False):
        H, W = input_size
        self.input_size, self.device, self.device_preproc = tuple(input_size), device, device_preproc
        self.host = torch.full((n, H, W, 3), 114, dtype=torch.uint8).pin_memory()
        self.dev = None

    def __call__(self, images):
        """images: n raw frames, None for an idle slot -> (frames [n,H,W,3], ratios, sizes (h, w)); None ratio and size for an idle
        slot, whose frame in the batch is stale.  Every NV12 frame is checked before any is letterboxed."""
        nv12 = [nv12_size(im) is not None for im in images]
        if self.dev is None and (self.device_preproc or any(nv12)):
            self.dev = torch.empty(self.host.shape, dtype=torch.uint8, device=self.device)
        lb = [None if im is None else letterbox_frame(im, self.input_size, self.device, self.host[i:i + 1],
                                                       None if self.dev is None else self.dev[i:i + 1], self.device_preproc)
              for i, im in enumerate(images)]
        if not any(t is not None and t[0].is_cuda for t in lb):
            frames = self.host
        else:
            frames = self.dev
            for i, t in enumerate(lb):
                if t is not None and not t[0].is_cuda:
                    frames[i:i + 1].copy_(t[0], non_blocking=True)
        return frames, [None if t is None else t[1] for t in lb], [None if t is None else t[2] for t in lb]


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


class UnicornSOTBatch:
    """`n_seq` SOT sequences in lock step: one batched frame (backbone -> interaction -> upsample -> correlation -> head -> NMS over
    all sequences) per step, captured as one CUDA graph.  Each sequence's results equal those of the same driver at n_seq = 1: every
    kernel of the batched frame computes each image as its B = 1 launch does.

    initialize(i, ...) sets sequence slot i at any time: its reference frame runs at B = 1 and its reference projection and label
    values are written in place into the static batched buffers the graphs read, so the graphs stay valid and the other slots are
    unaffected.  A slot that has not been initialised, or gets None in track(), computes on whatever its input buffer holds and its
    result is discarded.

    depth > 1: that many steps may be in flight (submit / collect), each on its own stream and engine context.  The frames of a
    sequence are independent — the network never sees the previous frame's result (unicorn_sot.py:57-109 uses only the initial
    frame's features and label map) — so overlapping them changes no output, only fills the SMs that one step's small kernels and
    launch gaps leave idle.  track() / track_tensor() stay synchronous (one step in, its result out).

    max_inst: detection rows read back per sequence; the greedy NMS scan stops there (the driver consumes output[:max_inst] only,
    unicorn_sot.py:69-70) unless full_nms=True, which computes the complete postprocess() list.  device_preproc: initialize() / track()
    upload the raw RGB frame and letterbox it on the GPU (uc_letterbox_u8, a bit-exact restatement of the reference's cv2 recipe).
    NV12 frames are always letterboxed on the GPU (letterbox_frame)."""

    def __init__(self, engine: UnicornEngine, input_size, n_seq, conf=0.001, nms=0.65, max_inst=3, use_graph=True, full_nms=False,
                 device_preproc=False, depth=1):
        assert n_seq >= 1 and depth >= 1
        self.eng, self.input_size, self.n_seq, self.depth = engine, tuple(input_size), n_seq, depth
        self.confthre, self.nmsthre, self.max_inst = conf, nms, max_inst
        self.nms_keep = 0 if full_nms else max_inst
        self.use_graph, self.device_preproc = use_graph, device_preproc
        H, W = self.input_size
        dev = engine.dev

        def make(eng, stream):  # a frame slot plus the pinned read-back of its counts and top max_inst rows
            s = FrameSlot(eng, H, W, stream, batch=n_seq)
            s.host_dets = torch.empty(n_seq, max_inst, 7, dtype=torch.float32).pin_memory()
            s.host_count = torch.zeros(n_seq, dtype=torch.int32).pin_memory()
            return s
        self._ring = Ring(in_flight(engine, depth, make))
        self._ctxs = self._ring.slots  # bench.py reads pipe._ctxs[i]
        self._ref_slot = FrameSlot(engine, H, W)  # B = 1 input of initialize
        n16 = (H // 16) * (W // 16)
        self.ref_proj = (torch.zeros(n_seq * n16, 256, dtype=torch.bfloat16, device=dev), torch.zeros(n_seq * n16, 256, dtype=torch.bfloat16, device=dev))
        self.lbs_pre = torch.zeros(n_seq, 1, (H // 8) * (W // 8), dtype=torch.float32, device=dev)
        self._frames = LetterboxBatch(n_seq, self.input_size, dev, device_preproc)  # the letterboxed frames of track()
        self.ready = [False] * n_seq
        self.states = [None] * n_seq
        self.launches_per_frame = 0  # bench.py reads it

    # slot 0 (tools/bench_batch.py replays its graph), and the intermediate tensors of the most recently collected step
    slot = property(lambda self: self._ctxs[0])
    last = property(lambda self: self._ctxs[(max(self._ring.collected, 1) - 1) % self.depth].last)

    # -------------------------------------------------------------------------------- device-side frame
    def _frame(self, c):
        e = c.eng
        e.begin_frame()
        values = self.lbs_pre if self.n_seq > 1 else self.lbs_pre[0]

        def correlate(seq):  # runs on a second stream while the neck runs on the main one
            f_pre, f_cur = e.interaction(None, seq["feat"], ref_proj=self.ref_proj)
            e_pre, e_cur = e.upsample(f_pre, "embp"), e.upsample(f_cur, "embc")
            return f_pre, f_cur, e_pre, e_cur, e.propagate(e_pre, e_cur, values)

        fpn, seq, (f_pre, f_cur, e_pre, e_cur, priors) = e.backbone(c.img, tag="cur", side=correlate)
        out = e.head(fpn, priors, "sot")
        ops.postprocess_device(out if self.n_seq > 1 else out[0], 1, self.confthre, self.nmsthre, c.ws, max_keep=self.nms_keep)
        c.last = dict(fpn=fpn, feat=seq["feat"], inter_pre=f_pre, inter_cur=f_cur, embed_pre=e_pre, embed_cur=e_cur, priors=priors, head=out)

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

    def submit(self, frames):
        """Pipelined protocol: enqueue a step (returns immediately); at most `depth` steps may be uncollected.  frames: [n_seq,H,W,3]
        uint8 or [n_seq,3,H,W] fp32 preprocessed, ideally pinned host memory.  On the slot's stream: input copy, graph replay (or eager
        launches), asynchronous read-back of (counts, top rows) into the slot's pinned buffers.  A slot's first graph step is warm-up,
        capture and replay in one call, so the graph exists after one step."""
        c = self._ring.submit()
        if c.stream is not None:  # the frames may have been written on the current stream
            c.stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(c.stream):  # None: the current stream
            c.stage(frames)
            if not self.use_graph:
                self._frame(c)
            elif c.graph is None:
                c.graph, self.launches_per_frame = c.capture(lambda: self._frame(c), warmup=True)
            else:
                c.graph.replay()
            c.host_count.copy_(c.ws.count, non_blocking=True)
            c.host_dets.copy_(c.ws.dets.view(self.n_seq, -1, 7)[:, :self.max_inst], non_blocking=True)
            c.event.record()

    def collect(self):
        """Result of the oldest submitted step: (dets [n_seq, max_inst, 7], counts [n_seq]) on the host; rows past a sequence's
        count are stale."""
        c = self._ring.collect()
        c.event.synchronize()
        return c.host_dets.clone(), c.host_count.clone()

    def track_tensor(self, frames):
        """submit + collect."""
        self.submit(frames)
        return self.collect()

    # -------------------------------------------------------------------------------- reference protocol
    def initialize(self, i, image, info: dict):
        """Slot i: image a raw frame, RGB uint8 [h, w, 3] or NV12 uint8 [3h/2, w] (letterbox_frame); info: init_bbox [x, y, w, h]."""
        ref, r, _ = letterbox_frame(image, self.input_size, self.eng.dev, device_preproc=self.device_preproc)
        self.initialize_tensor(i, ref, xyxy_resized(info["init_bbox"], r))
        self.states[i] = info["init_bbox"]

    def track(self, images):
        """images: n_seq raw frames, RGB uint8 [h, w, 3] or NV12 uint8 [3h/2, w] (letterbox_frame; the two may be mixed), None for an
        idle slot.  Returns n_seq results {"target_bbox": [x, y, w, h]}, None for idle or uninitialised slots."""
        assert len(images) == self.n_seq
        frames, ratios, _ = self._frames(images)
        dets, counts = self.track_tensor(frames)
        res = [None] * self.n_seq
        for i, r in enumerate(ratios):
            if r is None or not self.ready[i]:
                continue
            if int(counts[i]) > 0:
                self.states[i] = state_xywh(dets[i, 0], r, self.input_size)
            res[i] = {"target_bbox": self.states[i]}
        return res


class UnicornSOTTrack:
    """One SOT sequence: UnicornSOTBatch at n_seq = 1 (same arguments), under the reference's protocol.  Re-initialising writes the
    new reference in place, so the captured graphs are kept; steps still uncollected at initialize*() are forgotten."""

    def __init__(self, engine: UnicornEngine, input_size, conf=0.001, nms=0.65, max_inst=3, use_graph=True, full_nms=False,
                 device_preproc=False, depth=1):
        self._b = UnicornSOTBatch(engine, input_size, 1, conf, nms, max_inst, use_graph, full_nms, device_preproc, depth)
        self.state = None

    # what bench.py and the tests read: the driver's settings, its ring and slots, and slot 0's input buffer, graph and read-back
    eng = property(lambda self: self._b.eng)
    input_size = property(lambda self: self._b.input_size)
    max_inst = property(lambda self: self._b.max_inst)
    depth = property(lambda self: self._b.depth)
    launches_per_frame = property(lambda self: self._b.launches_per_frame)
    _ring = property(lambda self: self._b._ring)
    _ctxs = property(lambda self: self._b._ctxs)
    img_in_u8 = property(lambda self: self._b.slot.img_in_u8)
    graph = property(lambda self: self._b.slot.graph)
    host_dets = property(lambda self: self._b.slot.host_dets)
    last = property(lambda self: self._b.last)
    lbs_pre = property(lambda self: self._b.lbs_pre[0])  # fp32 [1, h8*w8], the values of a 2-D ops.corr_propagate

    def initialize_tensor(self, ref_frame, init_box_xyxy):
        """ref_frame: preprocessed fp32 [1,3,H,W] or uint8 [1,H,W,3] (host or device); init box in resized-image coordinates."""
        self._b.initialize_tensor(0, ref_frame, init_box_xyxy)
        self._b._ring.forget()

    def submit(self, cur_frame):
        """cur_frame: preprocessed fp32 [1,3,H,W] or uint8 [1,H,W,3], ideally pinned host memory."""
        self._b.submit(cur_frame)

    def collect(self):
        """Result of the oldest submitted frame: (dets[:max_inst] cpu, count)."""
        dets, count = self._b.collect()
        n = int(count[0])
        return dets[0, :min(n, self.max_inst)], n

    def track_tensor(self, cur_frame):
        self.submit(cur_frame)
        return self.collect()

    def initialize(self, image, info: dict):
        self._b.initialize(0, image, info)
        self._b._ring.forget()
        self.state = info["init_bbox"]

    def track(self, image, info: dict = None):
        self.state = self._b.track([image])[0]["target_bbox"]
        return {"target_bbox": self.state}

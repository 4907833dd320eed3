"""Frames in flight, shared by the per-frame drivers: a frame slot holds what one frame needs on the device (engine context, stream,
static input buffers, NMS workspace, CUDA graph, completion event), a ring hands the slots out in submission order."""
import torch

from . import _lib, ops


def anchor_count(H, W):
    """Head anchors of an H x W input: one per cell of the stride-8, 16 and 32 maps."""
    return (H // 8) * (W // 8) + (H // 16) * (W // 16) + (H // 32) * (W // 32)


class FrameSlot:
    """One frame in flight: the engine or engine fork (own activation buffers) it runs on, its stream (None: the current one), the
    two static input buffers a captured graph reads, the NMS workspace, the graph, a completion event and the frame's
    intermediate tensors (`last`).  batch > 1: the inputs hold that many frames and the workspace that many images."""

    def __init__(self, eng, H, W, stream=None, batch=1):
        dev = eng.dev
        self.eng, self.stream = eng, stream
        self.img_in = torch.empty(batch, 3, H, W, dtype=torch.float32, device=dev)   # PreprocessorX format
        self.img_in_u8 = torch.empty(batch, H, W, 3, dtype=torch.uint8, device=dev)  # letterboxed BGR frame: 4x fewer H2D bytes
        self.u8 = False
        self.ws = ops.PostWorkspace(anchor_count(H, W), dev, batch)
        self.graph = None
        self.event = torch.cuda.Event()
        self.last = {}

    @property
    def img(self):
        """The input buffer the frame reads."""
        return self.img_in_u8 if self.u8 else self.img_in

    def use_u8(self, u8):
        """Select the input buffer the frame reads (dropping a graph captured on the other one); returns it."""
        if u8 != self.u8:
            self.u8, self.graph = u8, None  # the captured graph reads the other buffer
        return self.img

    def stage(self, frame):
        """Copy fp32 [B,3,H,W] or uint8 [B,H,W,3] `frame` (host or device) into the matching static buffer; returns the buffer."""
        self.use_u8(frame.dtype == torch.uint8).copy_(frame, non_blocking=True)
        return self.img

    def capture(self, frame_fn, warmup=False):
        """Capture frame_fn() into a CUDA graph on this slot's stream and replay it once.  warmup=True first runs frame_fn() eagerly
        (buffer allocation, kernel attributes, plan-time autotuning); only for frames that may run twice.  Returns (graph, kernels
        it launches through the C ABI)."""
        if warmup:
            frame_fn()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        l0 = _lib.LAUNCHES
        with torch.cuda.graph(g, stream=self.stream):
            frame_fn()
        launches = _lib.LAUNCHES - l0
        g.replay()
        return g, launches


def in_flight(engine, depth, make):
    """`depth` slots made by make(engine, stream): depth 1 is one slot on `engine` and the current stream; otherwise slot 0 runs on
    `engine`, the others on forks of it, each on its own stream."""
    return [make(engine if i == 0 else engine.fork(), None if depth == 1 else torch.cuda.Stream(device=engine.dev))
            for i in range(depth)]


class Ring:
    """Submit / collect bookkeeping: submit() hands out the slot of the next frame, collect() the slot of the oldest uncollected one;
    at most len(slots) frames are uncollected."""

    def __init__(self, slots):
        self.slots, self.submitted, self.collected = slots, 0, 0

    def submit(self):
        assert self.submitted - self.collected < len(self.slots), "collect() a frame first"
        self.submitted += 1
        return self.slots[(self.submitted - 1) % len(self.slots)]

    def collect(self):
        assert self.collected < self.submitted, "nothing submitted"
        self.collected += 1
        return self.slots[(self.collected - 1) % len(self.slots)]

    def forget(self):
        """Forget the frames in flight: the next submit() hands out the first slot again."""
        self.submitted = self.collected = 0

    def reset(self):
        """forget() and drop every slot's graph (a new reference frame changes what the frame reads)."""
        self.forget()
        for s in self.slots:
            s.graph = None

"""Batched COCO detection: the image path of tools/test.py / tools/demo.py for the unicorn_det_* models (YOLOX + YOLOXHeadDet).

Each step takes up to `max_batch` images of any sizes, letterboxes them on the device into one batch (data_augment.py:194-214 preproc:
top-left placement, pad 114, BGR kept), then runs backbone -> neck -> head -> fused decode and score filter -> sort -> NMS as one CUDA
graph of max_batch images.  A partial batch runs in the same graph with idle slots: images never interact (every normalisation is per
image), so each image's rows are those of its own one-image run.  The rows are in network-input pixels, as postprocess() returns them;
unicorn_b200.results.coco_detections turns them into the evaluator's COCO dicts."""
import torch

from . import _lib, ops, post_ops
from .engine import STRIDES, UnicornEngine
from .frames import FrameSlot, Ring, anchor_count, in_flight


class UnicornDetector:
    """UnicornDetector(eng, input_size, max_batch, conf, nms, class_agnostic, use_graph, depth).

    detect(images) runs one step and returns, per image, (rows fp32 [n, 7] = x1, y1, x2, y2, obj, cls_conf, cls_id in input pixels, r).
    submit(images) / collect() split it: up to `depth` steps in flight, each on its own stream and engine context.
    Defaults are the COCO evaluator's: test_conf 0.01, nmsthre 0.65, class-aware NMS (tools/demo.py uses class_agnostic=True)."""

    def __init__(self, eng: UnicornEngine, input_size=(800, 1280), max_batch=1, conf=0.01, nms=0.65, class_agnostic=False, use_graph=True,
                 depth=1):
        H, W = input_size
        if eng.cfg["task"] != "det":
            raise ValueError(f"UnicornDetector: {eng.cfg_name} is not a detector config")
        if max_batch < 1 or depth < 1 or H % 32 or W % 32:
            raise ValueError(f"UnicornDetector: max_batch >= 1, depth >= 1 and an input size of multiples of 32 (got {max_batch}, {depth}, "
                             f"{tuple(input_size)})")
        self.eng, self.input_size, self.max_batch = eng, (H, W), max_batch
        self.conf, self.nms, self.class_agnostic, self.use_graph = conf, nms, class_agnostic, use_graph
        self.A = anchor_count(H, W)

        def make(e, stream):
            s = FrameSlot(e, H, W, stream, max_batch)
            s.use_u8(True)
            s.img_in_u8.fill_(114)
            s.warm = False
            return s
        self._ring = Ring(in_flight(eng, depth, make))
        self.launches_per_step = 0

    def _frame(self, c):
        e = c.eng
        e.begin_frame()
        fpn, _ = e.backbone(c.img, tag="det")
        e.head(fpn, None, "mot", decode=False)
        ro, cl, hw = e.head_maps
        post_ops.det_candidates(ro, cl, hw, STRIDES, e.ncls, self.conf, c.ws)
        post_ops.postprocess_nms(self.nms, c.ws, class_agnostic=self.class_agnostic)

    def submit(self, images, rgb=False):
        """images: list of 1..max_batch uint8 HWC images (numpy arrays or tensors, host or device), BGR as cv2 loads them (rgb=True:
        RGB).  Enqueues the step; returns immediately."""
        n = len(images)
        if not 1 <= n <= self.max_batch:
            raise ValueError(f"UnicornDetector: 1..{self.max_batch} images per step (got {n})")
        srcs = []
        for im in images:
            t = torch.as_tensor(im)
            if t.dtype != torch.uint8 or t.dim() != 3 or t.shape[2] != 3:
                raise ValueError(f"UnicornDetector: images must be uint8 [h, w, 3], got {tuple(t.shape)} {t.dtype}")
            srcs.append(t)
        c = self._ring.submit()
        if c.stream is not None:
            c.stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(c.stream):
            c.ratios = []
            c.n = n
            for i, t in enumerate(srcs):
                src = t.to(c.eng.dev, non_blocking=True).contiguous()
                c.last[i] = src  # the upload stays alive until the step is collected
                c.ratios.append(ops.letterbox_u8(src, self.input_size, swap_rb=rgb, out=c.img_in_u8[i:i + 1])[1])
            if c.graph is not None:
                c.graph.replay()
            elif self.use_graph:
                c.graph, self.launches_per_step = c.capture(lambda: self._frame(c), warmup=not c.warm)
            else:
                l0 = _lib.LAUNCHES
                self._frame(c)
                self.launches_per_step = _lib.LAUNCHES - l0
            c.warm = True
            c.count_host = c.ws.count.to("cpu", non_blocking=True)
            c.event.record()

    def collect(self):
        """Rows of the oldest submitted step: a list of (rows fp32 [n, 7] CPU tensor in descending score order, r), one per image."""
        c = self._ring.collect()
        c.event.synchronize()
        dets = c.ws.dets.view(self.max_batch, self.A, 7)
        out = [(dets[i, :int(c.count_host[i])].cpu(), c.ratios[i]) for i in range(c.n)]
        c.last.clear()
        return out

    def detect(self, images, rgb=False):
        """One step: submit(images) then collect()."""
        self.submit(images, rgb)
        return self.collect()

"""Batched COCO detection: the image path of tools/test.py / tools/demo.py for the unicorn_det_* models (YOLOX + YOLOXHeadDet).

Each step takes up to `max_batch` images of any sizes, letterboxes them on the device into one batch (data_augment.py:194-214 preproc:
top-left placement, pad 114, BGR kept), then runs backbone -> neck -> head -> fused decode and score filter -> sort -> NMS as one CUDA
graph of max_batch images.  A partial batch runs in the same graph with idle slots: images never interact (every normalisation is per
image), so each image's rows are those of its own one-image run.  The rows are in network-input pixels, as postprocess() returns them;
unicorn_b200.results.coco_detections turns them into the evaluator's COCO dicts."""
import torch

from . import _lib, post_ops
from .engine import STRIDES, UnicornEngine
from .frames import FrameSlot, Ring, anchor_count, in_flight
from .mots import MaskEncoder
from .sot import letterbox_frame, nv12_size


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

    with_masks = False  # the head also runs the controller convs (UnicornInstanceSegmenter)

    def _frame(self, c):
        e = c.eng
        e.begin_frame()
        fpn, _ = e.backbone(c.img, tag="det")
        e.head(fpn, None, "mot", decode=False, with_masks=self.with_masks)
        ro, cl, hw = e.head_maps
        post_ops.det_candidates(ro, cl, hw, STRIDES, e.ncls, self.conf, c.ws)
        post_ops.postprocess_nms(self.nms, c.ws, class_agnostic=self.class_agnostic)
        return fpn

    def submit(self, images, rgb=False):
        """images: list of 1..max_batch images (numpy arrays or tensors, host or device): uint8 HWC, BGR as cv2 loads them (rgb=True:
        RGB), or NV12 uint8 [3h/2, w], which always gives BGR (sot.letterbox_frame); the two may be mixed.  Enqueues the step; returns
        immediately."""
        n = len(images)
        if not 1 <= n <= self.max_batch:
            raise ValueError(f"UnicornDetector: 1..{self.max_batch} images per step (got {n})")
        srcs = []
        for im in images:
            t = torch.as_tensor(im)
            if nv12_size(t) is None and (t.dtype != torch.uint8 or t.dim() != 3 or t.shape[2] != 3):
                raise ValueError(f"UnicornDetector: images must be uint8 [h, w, 3], got {tuple(t.shape)} {t.dtype}")
            srcs.append(t)
        c = self._ring.submit()
        if c.stream is not None:
            c.stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(c.stream):
            c.ratios, c.sizes = [], []
            c.n = n
            for i, t in enumerate(srcs):
                _, r, size = letterbox_frame(t, self.input_size, c.eng.dev, device_out=c.img_in_u8[i:i + 1], device_preproc=True, rgb=rgb)
                c.ratios.append(r)
                c.sizes.append(size)
            if c.graph is not None:
                c.graph.replay()
            elif self.use_graph:
                c.graph, self.launches_per_step = c.capture(lambda: self._frame(c), warmup=not c.warm)
            else:
                l0 = _lib.LAUNCHES
                self._frame(c)
                self.launches_per_step = _lib.LAUNCHES - l0
            c.warm = True
            self._after_frame(c)
            c.count_host = c.ws.count.to("cpu", non_blocking=True)
            c.event.record()

    def _after_frame(self, c):
        """Work of a step that follows its graph (or eager frame) on the step's stream, before the counts are copied back."""

    def collect(self):
        """Rows of the oldest submitted step: a list of (rows fp32 [n, 7] CPU tensor in descending score order, r), one per image."""
        c = self._ring.collect()
        c.event.synchronize()
        dets = c.ws.dets.view(self.max_batch, self.A, 7)
        out = [(dets[i, :int(c.count_host[i])].cpu(), c.ratios[i]) for i in range(c.n)]
        return out

    def detect(self, images, rgb=False):
        """One step: submit(images) then collect()."""
        self.submit(images, rgb)
        return self.collect()


class UnicornInstanceSegmenter(UnicornDetector):
    """UnicornInstanceSegmenter(eng, input_size, max_batch, conf, nms, use_graph, depth, mask_thres, d_rate, chunk, capacity): the
    COCO instance segmenter (unicorn_inst_convnext_tiny: YOLOX + YOLOXHeadDetMask) on the letterbox, batching and submit / collect
    protocol of UnicornDetector, with class-aware NMS.

    collect() returns, per image, (rows fp32 [n, 7] as UnicornDetector gives them, r, rles): rles[i] is the COCO compressed RLE of row
    i's mask over the image's original h x w, as COCOInstEvaluator.convert_to_coco_format makes it (utils/boxes.py postprocess_inst:
    the dynamic-conv mask of every NMS row, aligned_bilinear x d_rate; then resized by 1/r and thresholded > mask_thres);
    unicorn_b200.results.coco_instances turns them into the evaluator's dicts.

    The masks of NMS rows are made `chunk` rows at a time (dynamic masks at 1/d_rate of the input, then uc_inst_encode_batched, which
    folds the final upsample into the resize, so the full-resolution masks are never stored).  The step's graph ends with the masks
    of rows [0, chunk); their encode follows it on the step's stream.  collect() reads the row counts and, while an image has more
    rows, runs the next chunk eagerly for all such images at once.  With seeded weights about 15000 rows per image survive NMS at
    conf 0.01 (DESIGN.md section 4.11): that is 150 chunks per image."""

    with_masks = True

    def __init__(self, eng: UnicornEngine, input_size=(800, 1280), max_batch=1, conf=0.01, nms=0.65, use_graph=True, depth=1, mask_thres=0.3,
                 d_rate=2, chunk=100, capacity=1 << 20):
        if eng.cfg["task"] != "det" or not eng.cfg["mask"]:
            raise ValueError(f"UnicornInstanceSegmenter: {eng.cfg_name} is not an instance-segmentation config")
        if d_rate != 2 or chunk < 1 or max_batch > 64 or max_batch * chunk > 65535:
            raise ValueError(f"UnicornInstanceSegmenter: d_rate 2 (the 144-channel up-mask layer upsamples x4), chunk >= 1, max_batch <= 64 "
                             f"and max_batch * chunk <= 65535 (got {d_rate}, {chunk}, {max_batch})")
        super().__init__(eng, input_size, max_batch, conf, nms, False, use_graph, depth)
        self.mask_thres, self.d_rate, self.chunk = mask_thres, d_rate, chunk
        for c in self._ring.slots:
            c.rows = RowMasks(max_batch, self.A, self.input_size, chunk, d_rate, mask_thres, eng.dev, capacity)

    def _frame(self, c):
        fpn = super()._frame(c)
        c.mf, c.um = c.eng.mask_branch(fpn)
        c.dyn = list(c.eng.dyn_levels)
        c.rows.masks(c.mf, c.um, c.dyn, c.ws, 0)

    def _after_frame(self, c):
        if c.n < self.max_batch:
            c.ws.count[c.n:].zero_()  # idle slots have no rows
        c.rows.enqueue(c.n, c.ws, c.ratios, c.sizes)

    def collect(self):
        """Rows and masks of the oldest submitted step: a list of (rows fp32 [n, 7] CPU tensor in descending score order, r, rles [n]),
        one per image."""
        c = self._ring.collect()
        with torch.cuda.stream(c.stream):
            c.event.synchronize()
            counts = [int(v) for v in c.count_host[:c.n]]
            rles = c.rows.strings(counts, c.mf, c.um, c.dyn, c.ws, c.ratios, c.sizes)
        dets = c.ws.dets.view(self.max_batch, self.A, 7)
        out = [(dets[i, :counts[i]].cpu(), c.ratios[i], rles[i]) for i in range(c.n)]
        return out


class RowMasks:
    """The masks of every NMS row of B images as COCO RLE strings over each image's original frame, `chunk` rows at a time (utils/
    boxes.py postprocess_inst: the dynamic-conv mask of every row, aligned_bilinear x d_rate, resized by 1/r, thresholded > thr).  Each
    chunk is dynamic_masks_rows at d_rate = 1 into `maps` [B, chunk, H/d_rate, W/d_rate], then uc_inst_encode_batched, which folds the
    final upsample into the resize, so the full-resolution masks are never stored.  Holds the buffers of one frame slot.

    masks(..., row0=0) may run inside the frame's CUDA graph; enqueue() queues the encode of rows [0, chunk) on the current stream, and
    strings() waits for it and runs the further chunks eagerly, one batch per chunk for all images that still have rows."""

    def __init__(self, B, A, input_size, chunk, d_rate, thr, device, capacity):
        H, W = input_size
        up, h, w = 8 // d_rate, H // 8, W // 8
        self.B, self.A, self.chunk, self.d_rate, self.thr, self.up = B, A, chunk, d_rate, thr, up
        self.image_of = torch.arange(B, dtype=torch.int32, device=device)
        self.maps = torch.empty(B, chunk, h * up, w * up, dtype=torch.float32, device=device)
        self.scratch = torch.empty(B * chunk * h * w, dtype=torch.float32, device=device)
        self.window = torch.zeros(B, dtype=torch.int32, device=device)  # each image's rows in the current chunk
        self.enc = MaskEncoder(B * chunk, device, capacity)

    def masks(self, mf, um, dyn, ws, row0):
        """The d_rate = 1 masks of NMS rows row0 .. row0 + chunk - 1 of every image into maps."""
        torch.sub(ws.count, row0, out=self.window).clamp_(0, self.chunk)
        anchors = ws.anchors.view(self.B, self.A)[:, row0:]
        post_ops.dynamic_masks_rows(mf, um, dyn, [(t.shape[1], t.shape[2]) for t in dyn], anchors, self.window, self.image_of, self.chunk,
                                    self.up, self.maps, self.scratch)

    def _encode(self, n, ws, row0, ratios, sizes):
        post_ops.inst_encode(self.maps[:n], ws.count, row0, self.d_rate, self.thr, ratios, [h for h, _ in sizes], [w for _, w in sizes],
                             self.enc.ws, self.enc.d_emit, self.enc.d_chars, self.enc.d_offsets)

    def enqueue(self, n, ws, ratios, sizes):
        """Queues the encode of the first n images' rows [0, chunk) (their masks are in maps) on the current stream; sizes: n original
        (h, w), ratios: their letterbox scales."""
        self.enc.reserve(max(h for h, _ in sizes), max(w for _, w in sizes))
        self.enc.enqueue(n * self.chunk, lambda: self._encode(n, ws, 0, ratios, sizes))

    def strings(self, counts, mf, um, dyn, ws, ratios, sizes):
        """After enqueue(): the strings of rows [0, counts[b]) of each of the n = len(counts) images, a list per image."""
        n, k = len(counts), self.chunk
        K = n * k
        flat = self.enc.strings(K, lambda: self._encode(n, ws, 0, ratios, sizes))
        rles = [flat[b * k:b * k + min(k, counts[b])] for b in range(n)]
        row0 = k
        while any(m > row0 for m in counts):
            self.masks(mf, um, dyn, ws, row0)
            run = lambda r=row0: self._encode(n, ws, r, ratios, sizes)  # noqa: E731
            self.enc.enqueue(K, run)
            flat = self.enc.strings(K, run)
            for b in range(n):
                rles[b] += flat[b * k:b * k + max(0, min(k, counts[b] - row0))]
            row0 += k
        return rles

"""MOTS per-frame driver (UNTESTED ON A GPU — written after the round-1 GPU budget was spent; see tests/test_mots_gpu.py):
the per-frame body of MOTEvaluator.evaluate_omni_mots (unicorn/evaluators/mot_evaluator.py:776-897) on the H100 engine:
whole-mode detector with the CondInst controllers -> NMS -> dynamic-conv masks of the kept detections -> embedding
sampling -> QuasiDenseEmbedTracker.match(return_index=True) -> masks of the tracked boxes in ascending-id order,
overlap free, area filter, RLE (results.mots_frame_result)."""
import torch
import torch.nn.functional as F

from . import ops
from .engine import UnicornEngine
from .frames import anchor_count
from .mot import QDEmbedding
from .results import mots_frame_result
from .tracker import QuasiDenseEmbedTracker


class UnicornMOTSTracker:
    def __init__(self, engine: UnicornEngine, input_size, conf=0.01, nms=0.7, score_thr=0.1, max_dets=64, mask_thres=0.3, d_rate=2,
                 min_box_area=100, tracker=None):
        assert engine.cfg["mask"], "MOTS needs a *_mask model"
        self.eng, self.input_size = engine, tuple(input_size)
        self.conf, self.nms, self.score_thr, self.max_dets = conf, nms, score_thr, max_dets
        self.mask_thres, self.d_rate, self.min_box_area = mask_thres, d_rate, min_box_area
        self.tracker = tracker or QuasiDenseEmbedTracker(device=engine.dev)
        H, W = self.input_size
        self.ws = ops.PostWorkspace(anchor_count(H, W), engine.dev)
        self.img_in = torch.empty(1, 3, H, W, dtype=torch.float32, device=engine.dev)
        self._qd = QDEmbedding(engine, H, W, max_dets, "mots.emb")
        self.frame_id = 0
        self.last = {}

    def step_tensor(self, frame, img_h, img_w):
        """frame: preprocessed fp32 [1,3,H,W]; (img_h, img_w): original image size.  Returns the tuple write_results_mots()
        consumes for this frame: (frame_id, ids (1-based), cat_id, img_h, img_w, rles)."""
        e = self.eng
        H, W = self.input_size
        self.frame_id += 1
        self.img_in.copy_(frame, non_blocking=True)
        e.begin_frame()
        fpn, seq = e.backbone(self.img_in, tag="mots%d" % (self.frame_id & 1))
        out = e.head(fpn, None, "mot", with_masks=True)
        dets, cnt = ops.postprocess_device(out[0], e.ncls, self.conf, self.nms, self.ws)
        mf, um = e.mask_branch(fpn)
        hw = [(t.shape[1], t.shape[2]) for t in e.dyn_levels]
        masks = ops.dynamic_masks(mf, um, e.dyn_levels, hw, self.ws, self.max_dets, up_rate=8 // self.d_rate, d_rate=self.d_rate)
        self._qd(e, seq["feat"], dets, cnt)  # pre_dict as in the MOT driver (:803-818)
        n = min(int(cnt.item()), self.max_dets)
        d, f = dets[:n].cpu(), self._qd.feats[:n].cpu()
        scale = min(H / float(img_h), W / float(img_w))
        # masks at the original image scale, thresholded (:804-805)
        m = F.interpolate(masks[:n, None], scale_factor=1 / scale, mode="bilinear", align_corners=False)[:, 0, :img_h, :img_w] > self.mask_thres
        scores = d[:, 4] * d[:, 5]
        keep = scores > self.score_thr
        boxes = torch.cat([d[keep, :4] / scale, scores[keep, None]], 1)
        m, f = m[keep.to(m.device)], f[keep]
        self.last = dict(dets=d, masks=masks[:n], head=out, mask_feats=mf, up_masks=um, dyn=[t for t in e.dyn_levels])
        if n == 0:  # outputs[0] is None: no tracking for this frame (mot_evaluator.py:803)
            return self.frame_id, [], 2, img_h, img_w, []
        ob, _, oid, idx = self.tracker.match(boxes, torch.ones(boxes.size(0)), f, self.frame_id, return_index=True)
        m = m[idx.to(m.device)]
        valid = oid > -1
        return mots_frame_result(self.frame_id, ob[valid], oid[valid], m[valid.to(m.device)].cpu(), img_h, img_w, self.min_box_area)

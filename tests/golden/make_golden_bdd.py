"""Golden fixture for the BDD100K MOT / MOTS test protocol: runs the UNMODIFIED reference loop
external/qdtrack/qdtrack/apis/test_omni.py:multi_gpu_test_omni on the CPU and records what it computes.

    python tests/golden/make_golden_bdd.py      (writes tests/golden/bdd_tiny_320.npz; build container only)

unicorn_track_tiny (MOT branch) and unicorn_track_tiny_mask (MOTS branch), seeded weights (make_state_dict), test size 320x320 from
288x320 originals (r = 1, as BDD100K's 720x1280 frames at 800x1280), N_FRAMES make_video frames quantised to uint8, one video each.

Only what is absent from the image or distributed is stubbed: mmcv (ProgressBar, runner.get_dist_info -> (0, 1)),
mmdet.core.bbox2result / encode_mask_results (mmdet 2.x behaviour; the mask "encode" keeps the binary mask because pycocotools
is absent, and so does pycocotools.mask.encode for encode_track_results), qdtrack.core (its own transforms files),
qdtrack.models.build_tracker (qdtrack's tracker file with mmdet's bbox_overlaps given as torchvision's box_iou), collect_results_cpu
(returns the rank's part), a wrapper that gives the model a `.module`, and mmdet-shaped data (identity img_norm_cfg).

Seeded weights score all but one detection below 0.08, so no track would start at the BDD init thresholds (0.4 MOT, 0.5 MOTS).
Both branches therefore run with the thresholds of LOWERED (recorded in the file as tracker_cfg_*): init and match thresholds in gaps
of the seeded scores and match confidences, obj below every score (so every row may match); every other tracker value is the
config's.  CONF is raised from the exp's 0.01 so that the masks of every detection fit the file; rows between CONF and
0.1 still reach the tracker (asserted).

Stored per branch (prefix mot_ / mots_), per frame f: the NMS rows (rows, rows_n), the embeddings the tracker got (feats, fp32), the
boxes, ids and labels it returned in its score order (tboxes, ids, labels, ids_n) and its duplicate mask (valids, per row), and the result dicts decomposed into arrays: bbox_result
per class (bbox_cls: class counts [F, 8]), track_results per class (MOT: track, track_cls, track_f64 = whether the frame's arrays are
float64), track_result dicts (MOTS: tr_id, tr_bbox, tr_label, tr_row = the NMS row whose mask it holds, tr_n), and every detection's
mask bit-packed in NMS order (masks) with the fraction of its pixels within 0.05 of the mask threshold (near_thr); the
detection-side decision margins (margins, see detection_margins)."""
import importlib.util
import json
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import ref_import  # noqa: E402
from unicorn_b200.weights import make_state_dict  # noqa: E402
from unicorn_b200.synthetic import make_video  # noqa: E402

QD = os.path.join(ref_import.REF_ROOT, "external", "qdtrack", "qdtrack")
H = W = 320
OH, OW = 288, 320
N_FRAMES, SEED, N_OBJ = 8, 3, 4
NCLS = 8
CONF, NMS = 0.03, 0.65
TRACKER = {  # configs/bdd100k/unicorn.py and configs/bdd100k_mots/segtrack-frcnn_r50_fpn_12e_bdd10k_fixed_pcan.py
    "mot": dict(init_score_thr=0.4, obj_score_thr=0.2, match_score_thr=0.5, memo_tracklet_frames=10, memo_backdrop_frames=1,
                memo_momentum=1.0, nms_conf_thr=0.5, nms_backdrop_iou_thr=0.3, nms_class_iou_thr=0.7, with_cats=True,
                match_metric="bisoftmax"),
    "mots": dict(init_score_thr=0.5, obj_score_thr=0.3, match_score_thr=0.5, memo_tracklet_frames=10, memo_backdrop_frames=1,
                 memo_momentum=1.0, nms_conf_thr=0.5, nms_backdrop_iou_thr=0.3, nms_class_iou_thr=0.7, with_cats=True,
                 match_metric="bisoftmax"),
}
LOWERED = dict(init_score_thr=0.0562, obj_score_thr=0.02, match_score_thr=0.47)
SCORE_MARGIN = 2e-3  # no score within this of init / obj, no match confidence within this of match / nms_conf
MASK_THR = 0.3  # test_omni.py: getattr(exp, "mask_thres", 0.3)


def _mod(name, pkg=False, **attrs):
    m = types.ModuleType(name)
    if pkg:
        m.__path__ = []
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    m = importlib.util.module_from_spec(spec)
    sys.modules[name] = m
    spec.loader.exec_module(m)
    return m


def bbox2result(bboxes, labels, num_classes):
    """mmdet 2.x mmdet/core/bbox/transforms.py bbox2result."""
    if bboxes.shape[0] == 0:
        return [np.zeros((0, 5), dtype=np.float32) for _ in range(num_classes)]
    if isinstance(bboxes, torch.Tensor):
        bboxes = bboxes.detach().cpu().numpy()
        labels = labels.detach().cpu().numpy()
    return [bboxes[labels == i, :] for i in range(num_classes)]


def encode_mask_results(mask_results):
    """mmdet 2.x encode_mask_results with the RLE encode replaced by keeping the binary mask."""
    return [[np.array(m, dtype=bool) for m in cls] for cls in mask_results]


class _Bar:
    def __init__(self, *a, **k):
        pass

    def update(self, *a, **k):
        pass


class _Registry:
    def register_module(self, *a, **k):
        return lambda cls: cls


class _Wrapped(torch.nn.Module):
    """What MMDistributedDataParallel gives test_omni: the model under `.module`."""

    def __init__(self, model):
        super().__init__()
        self.module = model

    def forward(self, *a, **k):
        return self.module(*a, **k)


LOG = []  # per match(): what the tracker got and returned
NMS_ROWS = []  # per frame: postprocess(_inst) rows (None: no detection)
PRED = []  # per frame: the head output postprocess(_inst) got, [A, 5 + NCLS] (cx, cy, w, h, obj, classes)
NEAR = []  # per frame (MOTS): per row, the fraction of its mask's pixels within 0.05 of the mask threshold


def install():
    ref_import.install()
    _mod("mmcv", pkg=True, ProgressBar=_Bar)
    _mod("mmcv.runner", get_dist_info=lambda: (0, 1))
    from torchvision.ops import box_iou
    _mod("mmdet", pkg=True)
    _mod("mmdet.core", bbox2result=bbox2result, encode_mask_results=encode_mask_results, bbox_overlaps=box_iou)
    sys.modules["pycocotools.mask"].encode = lambda a: [np.array(a[:, :, i], dtype=bool) for i in range(a.shape[2])]
    for name in ("qdtrack", "qdtrack.core", "qdtrack.core.track", "qdtrack.models", "qdtrack.models.trackers", "qdtrack.apis"):
        _mod(name, pkg=True)
    tr = _load("qdtrack.core.track.transforms", os.path.join(QD, "core", "track", "transforms.py"))
    sys.modules["qdtrack.core"].track2result = tr.track2result
    _load("qdtrack.core.track.transforms_mots", os.path.join(QD, "core", "track", "transforms_mots.py"))
    _mod("qdtrack.models.builder", TRACKERS=_Registry())
    qd = _load("qdtrack.models.trackers.quasi_dense_embed_tracker", os.path.join(QD, "models", "trackers", "quasi_dense_embed_tracker.py"))

    class Recording(qd.QuasiDenseEmbedTracker):
        def match(self, bboxes, labels, track_feats, frame_id, asso_tau=-1, return_index=False):
            conf = self._best_confs(bboxes, labels, track_feats)
            out = super().match(bboxes, labels, track_feats, frame_id, asso_tau, return_index=True)
            LOG.append(dict(frame_id=frame_id, bboxes=bboxes.clone(), feats=track_feats.clone(), ids=out[2].clone(), labels=out[1].clone(), tboxes=out[0].clone(),
                            valids=out[3].clone(), conf=conf))
            return out if return_index else out[:3]

        def _best_confs(self, bboxes, labels, feats):
            """The confidences the greedy assignment compares with match_score_thr / nms_conf_thr (the reference's loop, read only)."""
            if self.empty or bboxes.size(0) == 0:
                return []
            _, inds = bboxes[:, -1].sort(descending=True)
            b, lab, emb = bboxes[inds], labels[inds], feats[inds]
            ious = box_iou(b[:, :-1], b[:, :-1])
            keep = torch.ones(b.size(0), dtype=torch.bool)
            for i in range(1, b.size(0)):
                thr = self.nms_backdrop_iou_thr if b[i, -1] < self.obj_score_thr else self.nms_class_iou_thr
                keep[i] = not (ious[i, :i] > thr).any()
            b, lab, emb = b[keep], lab[keep], emb[keep]
            mb, ml, me, mi, _ = self.memo
            f = torch.mm(emb, me.t())
            s = (f.softmax(dim=1) + f.softmax(dim=0)) / 2
            s *= (lab.view(-1, 1) == ml.view(1, -1)).float()
            out = []
            for i in range(b.size(0)):
                c, j = torch.max(s[i, :], dim=0)
                out.append(float(c))
                if c > self.match_score_thr and mi[j] > -1 and b[i, -1] > self.obj_score_thr:
                    s[:i, j] = 0
                    s[i + 1:, j] = 0
            return out

    sys.modules["qdtrack.models"].build_tracker = lambda cfg: Recording(**{k: v for k, v in cfg.items() if k != "type"})
    mod = _load("qdtrack.apis.test_omni", os.path.join(QD, "apis", "test_omni.py"))
    mod.collect_results_cpu = lambda part, size, tmpdir=None: part
    mod.time = types.SimpleNamespace(sleep=lambda s: None)
    for fn in ("postprocess", "postprocess_inst"):
        orig = getattr(mod, fn)

        def rec(*a, __orig=orig, __inst=fn == "postprocess_inst", **k):
            PRED.append(a[0][0].clone())
            out = __orig(*a, **k)
            rows = out[0][0] if __inst else out[0]
            NMS_ROWS.append(None if rows is None else rows.clone())
            if __inst and rows is not None:  # the loop resizes by 1 / r = 1 (an identity) before the threshold
                NEAR.append(((out[1][0][:, 0, :OH, :OW] - MASK_THR).abs() < 0.05).float().mean(dim=(1, 2)))
            return out
        setattr(mod, fn, rec)
    return mod


def frames_u8():
    """The golden's frames: make_video at the original size, quantised to uint8, [N, OH, OW, 3] (channel order as given)."""
    f, _ = make_video(N_FRAMES, OH, OW, seed=SEED, n_obj=N_OBJ)
    return f.round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()


class _DC:
    def __init__(self, data):
        self.data = data


def loader(u8):
    norm = dict(mean=np.zeros(3, dtype=np.float32), std=np.ones(3, dtype=np.float32), to_rgb=False)
    items = []
    for t in range(u8.shape[0]):
        meta = dict(frame_id=t, ori_shape=(OH, OW, 3), img_norm_cfg=norm)
        items.append({"img_metas": [_DC([[meta]])], "img": [u8[t:t + 1].permute(0, 3, 1, 2).float()]})
    return items


class _Loader:
    def __init__(self, items):
        self.dataset = items

    def __iter__(self):
        return iter(self.dataset)


def run(mod, name, mots):
    exp, model = ref_import.get_model(name)
    print(name, model.load_state_dict(make_state_dict(name, 0), strict=True))
    exp.test_size, exp.test_conf, exp.nmsthre = (H, W), CONF, NMS
    assert exp.grid_sample and exp.num_classes == NCLS and getattr(exp, "use_raft", False) == mots
    cfg = dict(TRACKER["mots" if mots else "mot"], **LOWERED)
    LOG.clear()
    NMS_ROWS.clear()
    PRED.clear()
    NEAR.clear()
    items = loader(frames_u8())
    res = mod.multi_gpu_test_omni(_Wrapped(model), _Loader(items), exp, dict(type="QuasiDenseEmbedTracker", **cfg), mots=mots)
    return cfg, dict(res), list(NMS_ROWS), list(LOG)


def corners(p):
    return torch.stack([p[:, 0] - p[:, 2] / 2, p[:, 1] - p[:, 3] / 2, p[:, 0] + p[:, 2] / 2, p[:, 1] + p[:, 3] / 2], 1)


def nms_margins(pred, conf):
    """The decisions of postprocess on one frame's head output: (min |score - conf| over every anchor, min gap between the top two
    class probabilities of a candidate, min |IoU - NMS| between a kept candidate and a lower-scored one of its class)."""
    from torchvision.ops import box_iou
    cls, lab = pred[:, 5:5 + NCLS].topk(2, dim=1)
    score = pred[:, 4] * cls[:, 0]
    keep = score >= conf
    m_conf = (score - conf).abs().min().item()
    m_cls = ((cls[keep, 0] - cls[keep, 1]) * pred[keep, 4]).min().item() if keep.any() else 1.0
    b, s, lb = corners(pred[keep]), score[keep], lab[keep, 0]
    order = s.sort(descending=True)[1]
    b, lb = b[order], lb[order]
    iou = box_iou(b, b)
    alive = torch.ones(len(b), dtype=torch.bool)
    m_iou = 1.0
    for i in range(len(b)):  # greedy NMS: only a kept box's IoU decides
        if not alive[i]:
            continue
        later = torch.arange(len(b)) > i
        same = later & (lb == lb[i])
        if same.any():
            m_iou = min(m_iou, (iou[i, same] - NMS).abs().min().item())
        alive &= ~(same & (iou[i] > NMS))
    return m_conf, m_cls, m_iou


def dedup_margin(log, cfg):
    """min |IoU - thr| of the tracker's duplicate removal (each row against every higher-scored row)."""
    from torchvision.ops import box_iou
    m = 1.0
    for e in log:
        b = e["bboxes"][e["bboxes"][:, 4].sort(descending=True)[1]]
        if len(b) < 2:
            continue
        iou = box_iou(b[:, :4], b[:, :4])
        thr = torch.where(b[:, 4] < cfg["obj_score_thr"], cfg["nms_backdrop_iou_thr"], cfg["nms_class_iou_thr"])
        low = torch.tril(torch.ones_like(iou, dtype=torch.bool), diagonal=-1)
        m = min(m, (iou - thr[:, None]).abs()[low].min().item())
    return m


def detection_margins(cfg, log, preds):
    """The smallest distance of the detection-side decisions from their thresholds over all frames: the conf threshold, the top-two
    class gap, the NMS IoU and the tracker's duplicate-removal IoU.  Under this protocol they decide which rows enter the bisoftmax,
    so they are id decisions too.  The seeded weights' candidate scores are too dense for these to clear the engine's bf16 error
    (DESIGN.md section 4.13), so they are recorded, not asserted: the ids are pinned on the golden's own rows (the host half) and,
    end to end, on the rows the engine read back."""
    m = [nms_margins(p, CONF) for p in preds]
    return dict(conf=min(v[0] for v in m), cls=min(v[1] for v in m), nms_iou=min(v[2] for v in m), dedup_iou=dedup_margin(log, cfg))


def check_coverage(cfg, log, rows):
    """Tracks persist across frames in more than one class, rows below 0.1 reach the tracker, no tracker decision on the golden's
    rows is near its threshold."""
    assert all(r is not None for r in rows) and len(log) == N_FRAMES
    seen, persist = {}, set()
    for e in log:
        for tid, lab in zip(e["ids"].tolist(), e["labels"].tolist()):
            if tid > -1:
                if tid in seen:
                    persist.add(int(lab))
                seen[tid] = lab
    assert len(persist) >= 2, persist
    assert any(bool((e["bboxes"][:, 4] < 0.1).any()) for e in log)
    scores = torch.cat([e["bboxes"][:, 4] for e in log])
    for k in ("init_score_thr", "obj_score_thr"):
        m = (scores - cfg[k]).abs().min().item()
        assert m > SCORE_MARGIN, (k, m)
    conf = torch.tensor([c for e in log for c in e["conf"]])
    # nms_conf_thr decides only for rows below obj_score_thr
    for k in ("match_score_thr", "nms_conf_thr") if bool((scores < cfg["obj_score_thr"]).any()) else ("match_score_thr",):
        m = (conf - cfg[k]).abs().min().item()
        assert m > SCORE_MARGIN, (k, m)
    return sorted(persist), len(seen)


def pack(masks):
    return np.packbits(np.asarray(masks, dtype=bool).reshape(len(masks), -1), axis=1)


def main():
    mod = install()
    out = dict(size=np.array([H, W]), orig=np.array([OH, OW]), n_frames=N_FRAMES, seed_video=SEED, n_obj=N_OBJ, conf=CONF, nms=NMS,
               ncls=NCLS, tracker_bdd=json.dumps(TRACKER), lowered=json.dumps(LOWERED))
    for mots, p in ((False, "mot_"), (True, "mots_")):
        cfg, res, rows, log = run(mod, "unicorn_track_tiny_mask" if mots else "unicorn_track_tiny", mots)
        persist, n_ids = check_coverage(cfg, log, rows)
        margins = detection_margins(cfg, log, list(PRED))
        print(p, "detection-side decision margins", margins)
        out[p + "margins"] = json.dumps(margins)
        print(p, "rows per frame", [r.shape[0] for r in rows], "ids", n_ids, "classes that persist", persist,
              "rows < 0.1:", sum(int((e["bboxes"][:, 4] < 0.1).sum()) for e in log))
        out[p + "tracker_cfg"] = json.dumps(cfg)
        out[p + "rows"] = torch.cat(rows).numpy()
        out[p + "rows_n"] = np.array([r.shape[0] for r in rows])
        out[p + "feats"] = torch.cat([e["feats"] for e in log]).numpy()
        out[p + "ids"] = torch.cat([e["ids"] for e in log]).numpy()
        out[p + "labels"] = torch.cat([e["labels"] for e in log]).numpy()
        out[p + "ids_n"] = np.array([e["ids"].numel() for e in log])
        out[p + "tboxes"] = torch.cat([e["tboxes"] for e in log]).numpy()
        out[p + "valids"] = torch.cat([e["valids"] for e in log]).numpy()
        bkey = "bbox_result" if mots else "bbox_results"
        out[p + "bbox"] = np.concatenate([a for fr in res[bkey] for a in fr])
        out[p + "bbox_cls"] = np.array([[a.shape[0] for a in fr] for fr in res[bkey]])
        assert all(a.dtype == np.float32 for fr in res[bkey] for a in fr)
        if not mots:
            tr = res["track_results"]
            out[p + "track"] = np.concatenate([a.astype(np.float64) for fr in tr for a in fr])
            out[p + "track_cls"] = np.array([[a.shape[0] for a in fr] for fr in tr])
            out[p + "track_f64"] = np.array([fr[0].dtype == np.float64 for fr in tr])
            assert all(len({a.dtype for a in fr}) == 1 for fr in tr)
            continue
        masks, tr_id, tr_bbox, tr_label, tr_row, tr_n = [], [], [], [], [], []
        for f, fr in enumerate(res["segm_result"]):
            labels = rows[f][:, 6].numpy()
            per = [list(c) for c in fr]
            frame_masks = [per[int(lab)].pop(0) for lab in labels]  # every detection's mask back in NMS order
            assert all(not c for c in per)
            masks += frame_masks
            d = res["track_result"][f]
            tr_n.append(len(d))
            for tid, v in d.items():
                assert isinstance(tid, np.int64) and v["bbox"].dtype == np.float32 and v["label"].dtype == np.float32
                hit = [i for i, m in enumerate(frame_masks) if np.array_equal(m, v["segm"])]
                assert hit, (f, tid)
                tr_id.append(int(tid))
                tr_bbox.append(v["bbox"])
                tr_label.append(v["label"])
                tr_row.append(hit[0])
        assert masks[0].shape == (OH, OW)
        out[p + "masks"] = pack(masks)
        out[p + "near_thr"] = torch.cat(NEAR).numpy()
        assert len(out[p + "near_thr"]) == len(masks)
        out.update({p + "tr_id": np.array(tr_id, dtype=np.int64), p + "tr_bbox": np.array(tr_bbox, dtype=np.float32).reshape(-1, 5),
                    p + "tr_label": np.array(tr_label, dtype=np.float32), p + "tr_row": np.array(tr_row), p + "tr_n": np.array(tr_n)})
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "bdd_tiny_320.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()

"""Result formats of the MOT / MOTS evaluators (SURVEY.md 8(f) "next" row 2): the txt writers of
unicorn/evaluators/mot_evaluator.py:37-72, the overlap-free mask post-processing of :858-866 and the COCO run-length
encoding the MOTS writer stores (pycocotools.mask.encode on a Fortran-ordered mask, :884-888).

pycocotools is a third-party dependency of the reference that is absent from this image: `rle_encode` restates the
published COCO mask API (cocoapi/common/maskApi.c: rleEncode + rleToString — column-major run lengths starting with the
zero run, then 5 data bits per character with a continuation bit, chars offset by 48, counts after the second stored as
differences to the count two positions earlier).  Its parity is UNPINNED (no pycocotools here, no vectors in the reference);
tests check the round trip with `rle_decode` and a hand-computed example.

bbox2result / track2result / segtrack2result are the per-frame result builders of the BDD100K test loop (qdtrack's test_omni.py),
with the dtypes of mmdet and qdtrack."""
from collections import defaultdict

import numpy as np
import torch


def _fmt(v, nd):
    return round(float(v), nd)


def write_results(filename, results):
    """MOT-challenge txt (mot_evaluator.py:50-60): results = [(frame_id, tlwhs, track_ids, scores), ...]; rows with id < 0 skipped."""
    with open(filename, "w") as f:
        for frame_id, tlwhs, track_ids, scores in results:
            for (x1, y1, w, h), tid, s in zip(tlwhs, track_ids, scores):
                if tid < 0:
                    continue
                f.write(f"{frame_id},{tid},{_fmt(x1, 1)},{_fmt(y1, 1)},{_fmt(w, 1)},{_fmt(h, 1)},{_fmt(s, 2)},-1,-1,-1\n")


def write_results_no_score(filename, results):
    """mot_evaluator.py:63-72: results = [(frame_id, tlwhs, track_ids), ...]."""
    with open(filename, "w") as f:
        for frame_id, tlwhs, track_ids in results:
            for (x1, y1, w, h), tid in zip(tlwhs, track_ids):
                if tid < 0:
                    continue
                f.write(f"{frame_id},{tid},{_fmt(x1, 1)},{_fmt(y1, 1)},{_fmt(w, 1)},{_fmt(h, 1)},-1,-1,-1,-1\n")


def write_results_mots(filename, results):
    """MOTS txt (mot_evaluator.py:37-47): results = [(frame_id, track_ids, cat_id, H, W, rles), ...]; ids are offset by 2000."""
    with open(filename, "w") as f:
        for frame_id, track_ids, cat_id, H, W, rles in results:
            for tid, rle in zip(track_ids, rles):
                if tid < 0:
                    continue
                f.write(f"{frame_id} {2000 + tid} {cat_id} {H} {W} {rle}\n")


def overlap_free(masks):
    """mot_evaluator.py:858-866: instance n keeps only the pixels no earlier instance (ascending track id) claimed.
    masks: bool [N,H,W] tensor -> bool [N,H,W] (one cumulative OR instead of the reference's Python loop)."""
    if masks.size(0) == 0:
        return masks
    m = masks.bool()
    claimed_before = (torch.cumsum(m.to(torch.int32), 0) - m.to(torch.int32)) > 0
    return m & ~claimed_before


def rle_encode(mask):
    """COCO compressed RLE string of a binary mask [H,W] (what pycocotools.mask.encode(np.asfortranarray(m))["counts"] holds)."""
    flat = np.asarray(mask, dtype=bool).reshape(-1, order="F")
    change = np.flatnonzero(flat[1:] != flat[:-1]) + 1
    bounds = np.concatenate([[0], change, [flat.size]])
    counts = np.diff(bounds).tolist()
    if flat.size and flat[0]:
        counts = [0] + counts  # the first run counts zeros
    out = []
    for i, c in enumerate(counts):
        x = int(c) - (int(counts[i - 2]) if i > 2 else 0)
        more = True
        while more:
            ch = x & 0x1F
            x >>= 5
            more = (x != -1) if (ch & 0x10) else (x != 0)
            if more:
                ch |= 0x20
            out.append(chr(ch + 48))
    return "".join(out)


def rle_decode(s, H, W):
    """Inverse of rle_encode: compressed string -> bool [H,W]."""
    counts, p = [], 0
    while p < len(s):
        x, k, more = 0, 0, True
        while more:
            c = ord(s[p]) - 48
            x |= (c & 0x1F) << (5 * k)
            more = bool(c & 0x20)
            p += 1
            k += 1
            if not more and (c & 0x10):
                x |= -1 << (5 * k)
        if len(counts) > 2:
            x += counts[-2]
        counts.append(x)
    flat = np.zeros(H * W, dtype=bool)
    pos, val = 0, False
    for c in counts:
        flat[pos:pos + c] = val
        pos += c
        val = not val
    return flat.reshape(H, W, order="F")


def mots_frame_result(frame_id, boxes, ids, masks, img_h, img_w, min_box_area=100, cat_id=2):
    """Host half of one MOTS frame after association (mot_evaluator.py:846-897): boxes [n,5] (x1,y1,x2,y2,score) and ids [n]
    as returned by QuasiDenseEmbedTracker.match (valid ids only, any order), masks bool [n,H,W] in the same order.
    Sorts by ascending id, makes the masks overlap free in that order, drops boxes with area <= min_box_area, encodes the
    survivors and returns the tuple write_results_mots() consumes: (frame_id, ids + 1, cat_id, img_h, img_w, rles)."""
    ids = torch.as_tensor(ids).long()
    boxes = torch.as_tensor(boxes, dtype=torch.float32)
    order = ids.sort()[1]
    ids, boxes, masks = ids[order], boxes[order], masks[order]
    free = overlap_free(masks).cpu().numpy() if masks.size(0) else None
    out_ids, rles = [], []
    for i in range(boxes.size(0)):
        tid = int(ids[i])
        if tid < 0:
            continue
        x1, y1, x2, y2 = boxes[i, :4].tolist()
        if (x2 - x1) * (y2 - y1) > min_box_area:
            rles.append(rle_encode(free[i]))
            out_ids.append(tid + 1)  # 1-based ids for the MOTS files
    return frame_id, out_ids, cat_id, img_h, img_w, rles


def coco_detections(rows, r, image_id, class_ids):
    """COCOEvaluator.convert_to_coco_format (unicorn/evaluators/coco_evaluator.py:128-158) for one image: rows fp32 [n, 7] (postprocess
    output in network-input pixels), r = the letterbox scale min(H / h, W / w), class_ids = the dataset's COCO category id of each
    contiguous class.  Returns the evaluator's dicts: bbox xywh in original pixels, score = obj * cls_conf."""
    if rows is None:
        return []
    rows = torch.as_tensor(rows).cpu()
    bboxes = rows[:, 0:4].clone()
    bboxes /= r
    bboxes[:, 2] = bboxes[:, 2] - bboxes[:, 0]
    bboxes[:, 3] = bboxes[:, 3] - bboxes[:, 1]
    cls = rows[:, 6]
    scores = rows[:, 4] * rows[:, 5]
    return [{"image_id": int(image_id), "category_id": class_ids[int(cls[i])], "bbox": bboxes[i].numpy().tolist(),
             "score": scores[i].numpy().item(), "segmentation": []} for i in range(bboxes.shape[0])]


def coco_instances(rows, rles, r, img_h, img_w, image_id, class_ids, polygons=True):
    """COCOInstEvaluator.convert_to_coco_format (unicorn/evaluators/coco_inst_evaluator.py) for one image: rows fp32 [n, 7] and rles [n]
    as UnicornInstanceSegmenter.collect() returns them (the masks already resized to img_h x img_w and thresholded), r the letterbox
    scale.  bbox, score and category_id are those of coco_detections.  polygons=True: "segmentation" holds the contours
    cv2.findContours(RETR_TREE, CHAIN_APPROX_SIMPLE) finds in the mask, flattened, those with more than 4 coordinates, and an
    instance left with none is dropped, as in the evaluator.  polygons=False: "segmentation" is the compressed RLE
    {"size": [img_h, img_w], "counts": rle} (pycocotools' format), and instances with an empty mask are dropped."""
    dets = coco_detections(rows, r, image_id, class_ids)
    assert len(dets) == len(rles)
    out = []
    for d, rle in zip(dets, rles):
        m = rle_decode(rle, img_h, img_w)
        if polygons:
            import cv2
            contours, _ = cv2.findContours(np.ascontiguousarray(m, dtype=np.uint8), cv2.RETR_TREE, cv2.CHAIN_APPROX_SIMPLE)
            d["segmentation"] = [c for c in (ct.flatten().tolist() for ct in contours) if len(c) > 4]
            if not d["segmentation"]:
                continue
        else:
            if not m.any():
                continue
            d["segmentation"] = {"size": [int(img_h), int(img_w)], "counts": rle}
        out.append(d)
    return out


def rle_dict(rle, img_h, img_w):
    """The dict pycocotools.mask.encode returns for one mask: {"size": [h, w], "counts": compressed RLE bytes}."""
    return {"size": [int(img_h), int(img_w)], "counts": rle.encode("ascii")}


def bbox2result(bboxes, labels, num_classes):
    """mmdet's bbox2result: bboxes [n, 5] (x1, y1, x2, y2, score), labels [n] -> num_classes float32 arrays [k, 5], each class's rows
    in their input order; [0, 5] arrays when n = 0."""
    if bboxes.shape[0] == 0:
        return [np.zeros((0, 5), dtype=np.float32) for _ in range(num_classes)]
    bboxes, labels = torch.as_tensor(bboxes).cpu().numpy(), torch.as_tensor(labels).cpu().numpy()
    return [bboxes[labels == i, :] for i in range(num_classes)]


def track2result(bboxes, labels, ids, num_classes):
    """qdtrack's track2result (core/track/transforms.py): the rows of valid ids (> -1) per class as [id, x1, y1, x2, y2, score].  The
    int64 ids joined to the float32 boxes make float64 arrays; a frame without a valid id gives float32 [0, 6] arrays."""
    valid = ids > -1
    bboxes, labels, ids = bboxes[valid], labels[valid], ids[valid]
    if bboxes.shape[0] == 0:
        return [np.zeros((0, 6), dtype=np.float32) for _ in range(num_classes)]
    bboxes, labels, ids = bboxes.cpu().numpy(), labels.cpu().numpy(), ids.cpu().numpy()
    return [np.concatenate((ids[labels == i, None], bboxes[labels == i, :]), axis=1) for i in range(num_classes)]


def segtrack2result(bboxes, labels, segms, ids):
    """qdtrack's segtrack2result (core/track/transforms_mots.py): {id: {"bbox", "label", "segm"}} of the valid ids (> -1), in row
    order; ids are numpy int64 keys, bbox float32 [5], label a numpy scalar of the labels' dtype, segm as given."""
    valid = ids > -1
    bboxes, labels, ids = bboxes[valid].cpu().numpy(), labels[valid].cpu().numpy(), ids[valid].cpu().numpy()
    segms = [s for s, v in zip(segms, valid.tolist()) if v]
    out = defaultdict(list)
    for bbox, label, segm, tid in zip(bboxes, labels, segms, ids):
        out[tid] = dict(bbox=bbox, label=label, segm=segm)
    return out

"""Quasi-dense embedding tracker on the H100 path — same constructor and `match` signature as the reference's
unicorn/tracker/quasi_dense_embed_tracker.py (QuasiDenseEmbedTracker.match :137-212, update_memo :47-102).

Everything dense lives on the device: the tracklet memo (ids, boxes, embeddings, labels, last frame, velocity) and the backdrops are
device tensors that never travel; the pairwise IoU matrices (duplicate removal, backdrop NMS), the bi-softmax embedding similarity
E.M^T and the greedy row-max assignment with column zeroing (:188-199) are sm_90a kernels (uc_box_iou, uc_bisoftmax, uc_qd_assign).
The host keeps the bookkeeping only (which id sits in which memo row) and reads back one small tensor per frame: the assigned
ids, which the caller needs anyway.  Inputs may be CPU or CUDA tensors; outputs come back on the device of `bboxes`, labels in the
caller's dtype, like the reference (which only indexes what it is given)."""
import torch

from .. import ops
from ._stream import assoc_stream


class QuasiDenseEmbedTracker:
    def __init__(self, init_score_thr=0.8, obj_score_thr=0.5, match_score_thr=0.5, memo_tracklet_frames=30,
                 memo_backdrop_frames=1, memo_momentum=0.8, nms_conf_thr=0.5, nms_backdrop_iou_thr=0.3,
                 nms_class_iou_thr=0.7, with_cats=True, match_metric="bisoftmax", device="cuda"):
        assert 0 <= memo_momentum <= 1.0 and memo_tracklet_frames >= 0 and memo_backdrop_frames >= 0
        if match_metric != "bisoftmax":
            raise NotImplementedError("only the bisoftmax metric (the reference default) is implemented")
        self.init_score_thr, self.obj_score_thr, self.match_score_thr = init_score_thr, obj_score_thr, match_score_thr
        self.memo_tracklet_frames, self.memo_backdrop_frames, self.memo_momentum = memo_tracklet_frames, memo_backdrop_frames, memo_momentum
        self.nms_conf_thr, self.nms_backdrop_iou_thr, self.nms_class_iou_thr = nms_conf_thr, nms_backdrop_iou_thr, nms_class_iou_thr
        self.with_cats = with_cats
        self.dev = torch.device(device)
        self.num_tracklets = 0
        # tracklet memo, one row per live id (insertion order == the reference's dict order), on the device
        d = self.dev
        self.t_ids = torch.zeros(0, dtype=torch.long, device=d)
        self.t_box = torch.zeros(0, 5, device=d)
        self.t_emb = None
        self.t_lab = torch.zeros(0, device=d)
        self.t_last = torch.zeros(0, dtype=torch.long, device=d)
        self.t_vel = torch.zeros(0, 5, device=d)
        self.t_acc = torch.zeros(0, dtype=torch.long, device=d)
        self._ids_host = []  # host mirror of t_ids (bookkeeping only)
        self.backdrops = []  # newest first: (boxes, embeds, labels), device tensors

    @property
    def empty(self):
        return len(self._ids_host) == 0

    # ---------------------------------------------------------------------------------------------- match
    def match(self, bboxes, labels, track_feats, frame_id, asso_tau=-1, return_index=False):
        labels_in, out_dev = labels, bboxes.device
        # descending-score order on the host copy of the scores (N floats; CPU torch.sort like the reference)
        order = bboxes[:, -1].detach().cpu().float().sort(descending=True)[1]
        labels_in = labels_in[order.to(labels_in.device)]
        with torch.cuda.stream(assoc_stream(self.dev)):  # not behind the next frame's kernels on the main stream
            od = order.to(self.dev)
            bboxes = bboxes.detach().to(self.dev, torch.float32)[od].contiguous()
            labels = labels.detach().to(self.dev, torch.float32)[od].contiguous()
            embeds = track_feats.detach().to(self.dev, torch.float32)[od].contiguous()
            n = bboxes.size(0)
            # duplicate removal: a box is dropped if ANY higher-scored box (kept or not) overlaps it above its threshold
            valids = torch.ones(n, dtype=torch.bool, device=self.dev)
            if n > 1:
                iou = ops.box_iou(bboxes[:, :4], bboxes[:, :4])
                thr = torch.where(bboxes[:, -1] < self.obj_score_thr, self.nms_backdrop_iou_thr, self.nms_class_iou_thr)
                valids = ~torch.tril(iou > thr[:, None], diagonal=-1).any(dim=1)  # row i vs columns < i
                bboxes, labels, embeds = bboxes[valids].contiguous(), labels[valids].contiguous(), embeds[valids].contiguous()
            labels_in = labels_in[valids.to(labels_in.device)]
            n = bboxes.size(0)
            ids = torch.full((n,), -1, dtype=torch.long, device=self.dev)
            if n > 0 and not self.empty:
                m_emb = torch.cat([self.t_emb] + [b[1] for b in self.backdrops]).contiguous()
                m_lab = torch.cat([self.t_lab] + [b[2] for b in self.backdrops]).contiguous()
                m_ids = torch.cat([self.t_ids] + [torch.full((b[1].size(0),), -1, dtype=torch.long, device=self.dev) for b in self.backdrops]).contiguous()
                scores = ops.bisoftmax(embeds, m_emb, labels if self.with_cats else None, m_lab if self.with_cats else None)
                # greedy, in detection-score order; a claimed memo column is zeroed for everybody else
                ids = ops.qd_assign(scores, m_ids, bboxes, self.match_score_thr, self.obj_score_thr, self.nms_conf_thr)
            new = (ids == -1) & (bboxes[:, 4] > self.init_score_thr) if n > 0 else torch.zeros(0, dtype=torch.bool, device=self.dev)
            ids_host = ids.cpu()  # the one read-back of the frame (the caller gets the ids on the host anyway)
            new_host = new.cpu()
            n_new = int(new_host.sum())
            ids_host[new_host] = torch.arange(self.num_tracklets, self.num_tracklets + n_new, dtype=torch.long)
            ids = ids_host.to(self.dev)
            self.num_tracklets += n_new
            self._update_memo(ids, ids_host, bboxes, embeds, labels, frame_id)
        if return_index:
            return bboxes.to(out_dev), labels_in, ids_host.to(out_dev), valids.to(out_dev)
        return bboxes.to(out_dev), labels_in, ids_host.to(out_dev)

    # ---------------------------------------------------------------------------------------------- memo
    def _update_memo(self, ids, ids_host, bboxes, embeds, labels, frame_id):
        d = self.dev
        if self.t_emb is None:
            self.t_emb = torch.zeros(0, embeds.size(1), device=d)
        pos = {t: k for k, t in enumerate(self._ids_host)}
        add, rows, slots = [], [], []
        for r, tid in enumerate(ids_host.tolist()):
            if tid < 0:
                continue
            k = pos.get(tid)
            if k is None:
                add.append(r)
            else:
                rows.append(r)
                slots.append(k)
        if rows:  # every id occurs once per frame: the memo rows are updated together (same arithmetic as the per-track loop)
            r, k = torch.tensor(rows, dtype=torch.long, device=d), torch.tensor(slots, dtype=torch.long, device=d)
            vel = (bboxes[r] - self.t_box[k]) / (frame_id - self.t_last[k]).float()[:, None]
            self.t_box[k] = bboxes[r]
            self.t_emb[k] = (1 - self.memo_momentum) * self.t_emb[k] + self.memo_momentum * embeds[r]
            self.t_last[k] = frame_id
            self.t_lab[k] = labels[r]
            acc = self.t_acc[k].float()[:, None]
            self.t_vel[k] = (self.t_vel[k] * acc + vel) / (acc + 1)
            self.t_acc[k] += 1
        if add:
            a = torch.tensor(add, dtype=torch.long, device=d)
            self.t_ids = torch.cat([self.t_ids, ids[a]])
            self.t_box = torch.cat([self.t_box, bboxes[a]])
            self.t_emb = torch.cat([self.t_emb, embeds[a]])
            self.t_lab = torch.cat([self.t_lab, labels[a]])
            self.t_last = torch.cat([self.t_last, torch.full((len(add),), frame_id, dtype=torch.long, device=d)])
            self.t_vel = torch.cat([self.t_vel, torch.zeros(len(add), bboxes.size(1), device=d)])
            self.t_acc = torch.cat([self.t_acc, torch.zeros(len(add), dtype=torch.long, device=d)])
            self._ids_host += [int(ids_host[r]) for r in add]
        # backdrops: unmatched (-1) boxes not overlapped (> thr) by any earlier box of this frame
        bd = torch.nonzero(ids == -1, as_tuple=False).squeeze(1)
        if bd.numel():
            iou = ops.box_iou(bboxes[bd, :4].contiguous(), bboxes[:, :4].contiguous())
            col = torch.arange(bboxes.size(0), device=d)[None, :]
            hit = ((iou > self.nms_backdrop_iou_thr) & (col < bd[:, None])).any(dim=1)
            bd = bd[~hit]
        self.backdrops.insert(0, (bboxes[bd], embeds[bd], labels[bd]))
        alive = (frame_id - self.t_last) < self.memo_tracklet_frames
        alive_host = alive.cpu()
        if not bool(alive_host.all()):
            self.t_ids, self.t_box, self.t_emb, self.t_lab = self.t_ids[alive], self.t_box[alive], self.t_emb[alive], self.t_lab[alive]
            self.t_last, self.t_vel, self.t_acc = self.t_last[alive], self.t_vel[alive], self.t_acc[alive]
            self._ids_host = [t for t, ok in zip(self._ids_host, alive_host.tolist()) if ok]
        if len(self.backdrops) > self.memo_backdrop_frames:
            self.backdrops.pop()


# The tracker settings of the BDD100K test protocol (qdtrack's test_omni.py): configs/bdd100k/unicorn.py (MOT) and
# configs/bdd100k_mots/segtrack-frcnn_r50_fpn_12e_bdd10k_fixed_pcan.py (MOTS).
BDD_TRACKER = dict(init_score_thr=0.4, obj_score_thr=0.2, match_score_thr=0.5, memo_tracklet_frames=10, memo_backdrop_frames=1,
                   memo_momentum=1.0, nms_conf_thr=0.5, nms_backdrop_iou_thr=0.3, nms_class_iou_thr=0.7, with_cats=True,
                   match_metric="bisoftmax")
BDD_MOTS_TRACKER = dict(BDD_TRACKER, init_score_thr=0.5, obj_score_thr=0.3)


def bdd_tracker(mots=False, device="cuda"):
    """A QuasiDenseEmbedTracker with the BDD100K MOT (mots=False) or MOTS (mots=True) test settings."""
    return QuasiDenseEmbedTracker(**(BDD_MOTS_TRACKER if mots else BDD_TRACKER), device=device)

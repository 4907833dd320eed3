"""ByteTrack association on the H100 path — mirrors unicorn/tracker/byte_tracker.py (BYTETracker.update :161-296,
STrack :13-144), unicorn/tracker/matching.py (iou_distance :73-91, fuse_score :173-180, linear_assignment :39-50)
and unicorn/tracker/kalman_filter.py (:23-269), with the same `BYTETracker(args).update(output_results, img_info,
img_size)` entry point used by unicorn/evaluators/mot_evaluator.py:100-245 / tools/track.py.

Differences in form, not in behaviour: the Kalman state of all tracks is one struct-of-arrays updated with batched
numpy algebra; the IoU cost matrices come from the sm_90a kernel uc_box_iou (inclusive-pixel convention of
cython_bbox); the assignment is the same extended-cost Jonker-Volgenant problem that `lap.lapjv(extend_cost=True,
cost_limit=t)` solves, solved with scipy's linear_sum_assignment (lap is not installed offline — optimal cost is
identical, tie-breaking between equal-cost optima is unpinned, see DESIGN.md §5)."""
import numpy as np
import torch
from scipy.optimize import linear_sum_assignment

from .. import ops
from ._stream import assoc_stream

NEW, TRACKED, LOST, REMOVED = 0, 1, 2, 3
_STD_POS, _STD_VEL = 1.0 / 20, 1.0 / 160
_F = np.eye(8)
_F[:4, 4:] = np.eye(4)
_Hm = np.eye(4, 8)


def _kf_initiate(xyah):
    h = xyah[3]
    std = np.array([2 * _STD_POS * h, 2 * _STD_POS * h, 1e-2, 2 * _STD_POS * h, 10 * _STD_VEL * h, 10 * _STD_VEL * h, 1e-5, 10 * _STD_VEL * h])
    return np.r_[xyah, np.zeros(4)], np.diag(std ** 2)


def _kf_predict(mean, cov):
    """batched: mean [n,8], cov [n,8,8]"""
    h = mean[:, 3]
    std = np.stack([_STD_POS * h, _STD_POS * h, np.full_like(h, 1e-2), _STD_POS * h, _STD_VEL * h, _STD_VEL * h, np.full_like(h, 1e-5), _STD_VEL * h], 1)
    q = np.zeros_like(cov)
    idx = np.arange(8)
    q[:, idx, idx] = std ** 2
    return mean @ _F.T, _F @ cov @ _F.T + q


def _kf_update(mean, cov, xyah):
    h = mean[3]
    r = np.diag(np.array([_STD_POS * h, _STD_POS * h, 1e-1, _STD_POS * h]) ** 2)
    pm, pc = _Hm @ mean, _Hm @ cov @ _Hm.T + r
    k = np.linalg.solve(pc, (cov @ _Hm.T).T).T  # pc is SPD: same solution as the reference's Cholesky solve
    innov = xyah - pm
    return mean + innov @ k.T, cov - k @ pc @ k.T


def _kf_update_batch(mean, cov, z):
    """_kf_update for n tracks at once: mean [n,8], cov [n,8,8], z [n,4] (H = [I4 | 0] selects, so H m and H P H^T are slices)."""
    h = mean[:, 3]
    r = np.zeros((len(h), 4, 4))
    idx = np.arange(4)
    r[:, idx, idx] = np.stack([_STD_POS * h, _STD_POS * h, np.full_like(h, 1e-1), _STD_POS * h], 1) ** 2
    pc = cov[:, :4, :4] + r
    k = np.linalg.solve(pc, cov[:, :, :4].transpose(0, 2, 1)).transpose(0, 2, 1)  # [n,8,4]
    innov = z - mean[:, :4]
    return mean + np.einsum("ni,nji->nj", innov, k), cov - k @ pc @ k.transpose(0, 2, 1)


def _update_matched(pairs, frame_id):
    """STrack.update for every (track, detection) pair of one association stage with ONE batched Kalman update."""
    if not pairs:
        return
    mean = np.stack([t.mean for t, _ in pairs])
    cov = np.stack([t.cov for t, _ in pairs])
    z = np.stack([t.xyah(d.tlwh) for t, d in pairs])
    mean, cov = _kf_update_batch(mean, cov, z)
    for i, (t, d) in enumerate(pairs):
        t.mean, t.cov = mean[i], cov[i]
        t.tracklet_len = 0 if t.state != TRACKED else t.tracklet_len + 1  # re-activation of a lost track restarts the length
        t.state, t.is_activated, t.frame_id, t.score = TRACKED, True, frame_id, d.score


class STrack:
    _count = 0  # process-wide id counter like BaseTrack._count (basetrack.py:13,34-37)

    def __init__(self, tlwh, score):
        self._tlwh = np.asarray(tlwh, dtype=np.float64)
        self.mean = self.cov = None
        self.is_activated = False
        self.score = score
        self.tracklet_len = 0
        self.state = NEW
        self.track_id = 0
        self.frame_id = self.start_frame = 0

    @staticmethod
    def next_id():
        STrack._count += 1
        return STrack._count

    @property
    def end_frame(self):
        return self.frame_id

    @property
    def tlwh(self):
        if self.mean is None:
            return self._tlwh.copy()
        r = self.mean[:4].copy()
        r[2] *= r[3]
        r[:2] -= r[2:] / 2
        return r

    @property
    def tlbr(self):
        r = self.tlwh
        r[2:] += r[:2]
        return r

    def xyah(self, tlwh=None):
        r = (self.tlwh if tlwh is None else np.asarray(tlwh, dtype=np.float64)).copy()
        r[:2] += r[2:] / 2
        r[2] /= r[3]
        return r

    def activate(self, frame_id):
        self.track_id = self.next_id()
        self.mean, self.cov = _kf_initiate(self.xyah(self._tlwh))
        self.tracklet_len, self.state = 0, TRACKED
        self.is_activated = frame_id == 1
        self.frame_id = self.start_frame = frame_id

    def update(self, det, frame_id, reactivate=False):
        self.mean, self.cov = _kf_update(self.mean, self.cov, self.xyah(det.tlwh))
        self.tracklet_len = 0 if reactivate else self.tracklet_len + 1
        self.state, self.is_activated, self.frame_id, self.score = TRACKED, True, frame_id, det.score


def _predict_all(tracks):
    if not tracks:
        return
    mean = np.stack([t.mean.copy() for t in tracks])
    cov = np.stack([t.cov for t in tracks])
    for i, t in enumerate(tracks):
        if t.state != TRACKED:
            mean[i, 7] = 0
    mean, cov = _kf_predict(mean, cov)
    for i, t in enumerate(tracks):
        t.mean, t.cov = mean[i], cov[i]


def _tlbr_all(tracks):
    """np.stack([t.tlbr for t in tracks]) without the per-track property calls (same arithmetic, same rounding)."""
    out = np.empty((len(tracks), 4))
    kf = [i for i, t in enumerate(tracks) if t.mean is not None]
    raw = [i for i, t in enumerate(tracks) if t.mean is None]
    if kf:
        r = np.stack([tracks[i].mean[:4] for i in kf])  # (cx, cy, a, h)
        w = r[:, 2] * r[:, 3]
        x, y = r[:, 0] - w / 2, r[:, 1] - r[:, 3] / 2
        out[kf] = np.stack([x, y, w + x, r[:, 3] + y], 1)
    if raw:
        r = np.stack([tracks[i]._tlwh for i in raw])
        out[raw] = np.concatenate([r[:, :2], r[:, 2:] + r[:, :2]], 1)
    return out


def iou_distance(a_tracks, b_tracks, device):
    if not a_tracks or not b_tracks:
        return np.zeros((len(a_tracks), len(b_tracks)))
    with torch.cuda.stream(assoc_stream(device)):  # not behind the next frame's kernels on the main stream
        a = torch.tensor(_tlbr_all(a_tracks), dtype=torch.float32, device=device)
        b = torch.tensor(_tlbr_all(b_tracks), dtype=torch.float32, device=device)
        return 1.0 - ops.box_iou(a, b, plus_one=True).cpu().numpy().astype(np.float64)


def fuse_score(cost, dets):
    if cost.size == 0:
        return cost
    return 1.0 - (1.0 - cost) * np.array([d.score for d in dets])[None, :]


def linear_assignment(cost, thresh):
    """lap.lapjv(cost, extend_cost=True, cost_limit=thresh): pairs costlier than thresh stay unmatched."""
    n, m = cost.shape
    if cost.size == 0:
        return np.empty((0, 2), dtype=int), list(range(n)), list(range(m))
    ext = np.full((n + m, n + m), thresh / 2.0)
    ext[n:, m:] = 0
    ext[:n, :m] = cost
    rows, cols = linear_sum_assignment(ext)
    matches = [(r, c) for r, c in zip(rows, cols) if r < n and c < m]
    mr, mc = {r for r, _ in matches}, {c for _, c in matches}
    return np.asarray(matches, dtype=int).reshape(-1, 2), [i for i in range(n) if i not in mr], [j for j in range(m) if j not in mc]


def _join(a, b):
    seen = {t.track_id for t in a}
    return a + [t for t in b if t.track_id not in seen and not seen.add(t.track_id)]


def _sub(a, b):
    drop = {t.track_id for t in b}
    return [t for t in a if t.track_id not in drop]


class BYTETracker:
    def __init__(self, args, frame_rate=30, device="cuda"):
        self.args = args
        self.device = device
        self.tracked, self.lost, self.removed = [], [], []
        self.frame_id = 0
        self.det_thresh = args.track_thresh + 0.1
        self.max_time_lost = int(frame_rate / 30.0 * args.track_buffer)

    def update(self, output_results, img_info, img_size):
        self.frame_id += 1
        out = output_results.detach().cpu().numpy() if torch.is_tensor(output_results) else np.asarray(output_results)
        if out.shape[1] == 5:
            scores, boxes = out[:, 4], out[:, :4].copy()
        else:
            scores, boxes = out[:, 4] * out[:, 5], out[:, :4].copy()
        boxes = boxes / min(img_size[0] / float(img_info[0]), img_size[1] / float(img_info[1]))
        hi = scores > self.args.track_thresh
        lo = (scores > 0.1) & (scores < self.args.track_thresh)
        def mk(bs, ss):  # tlbr -> tlwh for all detections at once
            tlwh = np.concatenate([bs[:, :2], bs[:, 2:] - bs[:, :2]], 1)
            return [STrack(t, s) for t, s in zip(tlwh, ss)]
        dets, dets2 = mk(boxes[hi], scores[hi]), mk(boxes[lo], scores[lo])
        activated, refound, lost, removed = [], [], [], []
        unconfirmed = [t for t in self.tracked if not t.is_activated]
        confirmed = [t for t in self.tracked if t.is_activated]
        pool = _join(confirmed, self.lost)
        _predict_all(pool)
        # first association: high-score detections, IoU x score
        d = iou_distance(pool, dets, self.device)
        if not getattr(self.args, "mot20", False):
            d = fuse_score(d, dets)
        m, u_trk, u_det = linear_assignment(d, self.args.match_thresh)
        for it, _ in m:
            (activated if pool[it].state == TRACKED else refound).append(pool[it])
        _update_matched([(pool[it], dets[idt]) for it, idt in m], self.frame_id)
        # second association: low-score detections against the still-tracked leftovers, plain IoU
        rest = [pool[i] for i in u_trk if pool[i].state == TRACKED]
        m, u_trk2, _ = linear_assignment(iou_distance(rest, dets2, self.device), 0.5)
        for it, _ in m:
            (activated if rest[it].state == TRACKED else refound).append(rest[it])
        _update_matched([(rest[it], dets2[idt]) for it, idt in m], self.frame_id)
        for it in u_trk2:
            if rest[it].state != LOST:
                rest[it].state = LOST; lost.append(rest[it])
        # unconfirmed tracks (one frame old) against the remaining high-score detections
        dets_left = [dets[i] for i in u_det]
        d = iou_distance(unconfirmed, dets_left, self.device)
        if not getattr(self.args, "mot20", False):
            d = fuse_score(d, dets_left)
        m, u_unc, u_det = linear_assignment(d, 0.7)
        activated.extend(unconfirmed[it] for it, _ in m)
        _update_matched([(unconfirmed[it], dets_left[idt]) for it, idt in m], self.frame_id)
        for it in u_unc:
            unconfirmed[it].state = REMOVED; removed.append(unconfirmed[it])
        for i in u_det:  # new tracks
            if dets_left[i].score >= self.det_thresh:
                dets_left[i].activate(self.frame_id); activated.append(dets_left[i])
        for t in self.lost:
            if self.frame_id - t.end_frame > self.max_time_lost:
                t.state = REMOVED; removed.append(t)
        self.tracked = _join(_join([t for t in self.tracked if t.state == TRACKED], activated), refound)
        self.lost = _sub(_sub(self.lost, self.tracked) + lost, self.removed)
        self.removed.extend(removed)
        # duplicates between tracked and lost (IoU distance < 0.15): keep the older track
        pd = iou_distance(self.tracked, self.lost, self.device)
        da, db = set(), set()
        for p, q in zip(*np.where(pd < 0.15)):
            tp = self.tracked[p].frame_id - self.tracked[p].start_frame
            tq = self.lost[q].frame_id - self.lost[q].start_frame
            (db if tp > tq else da).add(int(q) if tp > tq else int(p))
        self.tracked = [t for i, t in enumerate(self.tracked) if i not in da]
        self.lost = [t for i, t in enumerate(self.lost) if i not in db]
        return [t for t in self.tracked if t.is_activated]

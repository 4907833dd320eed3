"""MOT association on the GPU path against the oracle (and through it the reference): embedding sampling, the
quasi-dense tracker's ids over a 25-frame sequence (bit-matching track assignments), and the MOT driver."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))


def test_sample_embed_matches_grid_sample():
    import tracker_oracle as to
    from unicorn_b200 import ops
    g = torch.Generator().manual_seed(0)
    emb = torch.randn(1, 128, 20, 36, generator=g)
    boxes = torch.rand(40, 4, generator=g) * torch.tensor([288.0, 160.0, 288.0, 160.0])
    boxes[:, 2:] += boxes[:, :2]
    boxes[0] = torch.tensor([-50.0, -20.0, 4.0, 6.0])       # centre clamps to the border
    boxes[1] = torch.tensor([280.0, 150.0, 400.0, 300.0])
    ref = to.sample_embeddings(emb, boxes, (160, 288))
    e16 = emb[0].permute(1, 2, 0).contiguous().half().cuda().unsqueeze(0)
    cnt = torch.tensor([37], dtype=torch.int32, device="cuda")
    got = ops.sample_embed(e16, boxes.cuda().contiguous(), 40, 8.0, count=cnt).cpu()
    ref16 = to.sample_embeddings(emb.half().float(), boxes, (160, 288))
    assert torch.allclose(got[:37], ref16[:37], atol=2e-3), (got[:37] - ref16[:37]).abs().max()
    assert (got[37:] == 0).all()
    assert (got[:37] - ref[:37]).abs().max() < 2e-2


def test_bisoftmax_and_iou_kernels():
    import tracker_oracle as to
    from unicorn_b200 import ops
    g = torch.Generator().manual_seed(1)
    E, M = torch.randn(23, 128, generator=g), torch.randn(57, 128, generator=g)
    le, lm = torch.randint(0, 3, (23,), generator=g).float(), torch.randint(0, 3, (57,), generator=g).float()
    f = E @ M.t()
    ref = (f.softmax(1) + f.softmax(0)) / 2 * (le[:, None] == lm[None, :]).float()
    got = ops.bisoftmax(E.cuda(), M.cuda(), le.cuda(), lm.cuda()).cpu()
    assert torch.allclose(got, ref, atol=1e-5, rtol=1e-4)
    a = torch.rand(31, 4, generator=g) * 100
    a[:, 2:] += a[:, :2]
    b = torch.rand(17, 4, generator=g) * 100
    b[:, 2:] += b[:, :2]
    assert torch.allclose(ops.box_iou(a.cuda(), b.cuda()).cpu(), to.box_iou(a, b), atol=1e-6)


def test_qd_tracker_ids_match_reference():
    from unicorn_b200.synthetic import make_detections
    from unicorn_b200.tracker import QuasiDenseEmbedTracker
    g = np.load(os.path.join(ROOT, "tests", "golden", "qd_tracker.npz"))
    frames = make_detections(int(g["n_frames"]), int(g["n_obj"]), int(g["seed"]))
    trk = QuasiDenseEmbedTracker()
    for i, (boxes, feats) in enumerate(frames):
        b, _, ids = trk.match(boxes, torch.ones(boxes.size(0)), feats, i + 1)
        assert np.array_equal(ids.numpy(), g[f"ids_{i}"]), (i, ids, g[f"ids_{i}"])
        assert np.allclose(b.numpy(), g[f"boxes_{i}"])
    # SURVEY 8(f3): the memo never leaves the device, the greedy assignment is a kernel (uc_qd_assign)
    assert trk.t_emb.is_cuda and trk.t_box.is_cuda and all(t.is_cuda for bd in trk.backdrops for t in bd)
    assert trk.num_tracklets == int(g["num_tracklets"])


def test_qd_assign_kernel_matches_reference_loop():
    """uc_qd_assign against the reference's loop (quasi_dense_embed_tracker.py:188-199) on random score matrices with ties, claimed
    columns, backdrop columns and the three thresholds in play."""
    from unicorn_b200 import ops
    g = torch.Generator().manual_seed(7)
    for N, M in ((1, 1), (17, 5), (40, 90), (300, 700)):
        sc = torch.rand(N, M, generator=g)
        sc[sc < 0.3] = 0.0
        sc[:, M // 3] = sc[:, 0]  # exact ties between columns: the first maximum wins
        memo_ids = torch.randint(-1, 50, (M,), generator=g)
        boxes = torch.rand(N, 5, generator=g)
        ref, s2 = torch.full((N,), -1, dtype=torch.long), sc.clone()
        for i in range(N):
            conf, j = torch.max(s2[i], dim=0)
            if conf > 0.5 and memo_ids[j] > -1:
                if boxes[i, 4] > 0.5:
                    ref[i] = memo_ids[j]
                    s2[:i, j] = 0
                    s2[i + 1:, j] = 0
                elif conf > 0.6:
                    ref[i] = -2
        got = ops.qd_assign(sc.cuda().contiguous(), memo_ids.cuda(), boxes.cuda().contiguous(), 0.5, 0.5, 0.6).cpu()
        assert torch.equal(got, ref), (N, M)


def test_mot_driver_runs_and_is_consistent():
    """tiny model, 4 frames, 3 moving objects: whole mode + interaction + sampling + association end to end; the
    sampled embeddings are checked against the oracle's grid_sample on the engine's own embedding map."""
    import tracker_oracle as to
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.mot import UnicornMOTTracker
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.weights import make_state_dict
    name = "unicorn_track_tiny"
    eng = UnicornEngine(make_state_dict(name, 0), name)
    frames, _ = make_video(4, 320, 320, seed=1, n_obj=3)
    from unicorn_b200.tracker import QuasiDenseEmbedTracker
    # seeded random weights give low scores: lower the tracker's score gates so that tracklets are created
    mot = UnicornMOTTracker(eng, (320, 320), conf=0.01, nms=0.7, score_thr=0.02,
                            tracker=QuasiDenseEmbedTracker(init_score_thr=0.05, obj_score_thr=0.03))
    all_ids = []
    for t in range(4):
        boxes, ids = mot.step_tensor(frames[t:t + 1])
        all_ids.append(ids)
        d, f = mot.last["dets"], mot.last["feats"]
        assert d.shape[0] > 0
        emb = mot.last["embed"].float().permute(0, 3, 1, 2).cpu()
        ref = to.sample_embeddings(emb, d[:, :4], (320, 320))
        assert torch.allclose(f, ref, atol=2e-3), (f - ref).abs().max()
        assert (ids >= 0).all() and ids.numel() == ids.unique().numel()
    assert mot.tracker.num_tracklets >= 1


def test_mot_pipelined_graph_matches_sequential():
    """submit(t+1) before collect(t), device half replayed from CUDA graphs: identical detections, embeddings and track
    ids as the sequential eager protocol (nothing on the device depends on the association)."""
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.mot import UnicornMOTTracker
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.tracker import QuasiDenseEmbedTracker
    from unicorn_b200.weights import make_state_dict
    name = "unicorn_track_tiny"
    eng = UnicornEngine(make_state_dict(name, 0), name)
    frames, _ = make_video(7, 320, 320, seed=2, n_obj=3)
    mk = lambda **kw: UnicornMOTTracker(eng, (320, 320), conf=0.01, nms=0.7, score_thr=0.02,  # noqa: E731
                                        tracker=QuasiDenseEmbedTracker(init_score_thr=0.05, obj_score_thr=0.03), **kw)
    seq = mk()
    ref = []
    for t in range(7):
        b, i = seq.step_tensor(frames[t:t + 1])
        ref.append((b.clone(), i.clone(), seq.last["dets"].clone(), seq.last["feats"].clone()))
    pipe = mk(use_graph=True)
    got = []
    pipe.submit(frames[0:1])
    for t in range(7):
        if t + 1 < 7:
            pipe.submit(frames[t + 1:t + 2])
        b, i = pipe.collect()
        got.append((b.clone(), i.clone(), pipe.last["dets"].clone(), pipe.last["feats"].clone()))
    assert len(pipe._graphs) == 2
    for t, (r, g) in enumerate(zip(ref, got)):
        assert torch.equal(r[2], g[2]), f"frame {t}: detections differ"
        assert torch.equal(r[3], g[3]), f"frame {t}: embeddings differ"
        assert torch.equal(r[1], g[1]) and torch.equal(r[0], g[0]), f"frame {t}: tracks differ"


def test_mot_byte_arm_three_frames_in_flight_matches_one_stream():
    """ByteTrack arm (mot_evaluator.py:177-209): with depth=3 the device halves of three frames run on their own streams / engine
    contexts (CUDA graphs from a context's second frame on); the detection rows handed to BYTETracker.update per frame must be
    bit-identical to the one-stream driver's, in frame order (the tracker itself is checked in test_byte_tracker_matches_reference_logic)."""
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.mot import UnicornMOTTracker
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.weights import make_state_dict

    class Recorder:  # stands in for BYTETracker: update(dets [n,7] numpy, img_info, img_size)
        def __init__(self):
            self.rows = []

        def update(self, dets, img_info, img_size):
            self.rows.append(torch.from_numpy(dets).clone())
            return []
    name = "unicorn_track_tiny"
    eng = UnicornEngine(make_state_dict(name, 0), name)
    frames, _ = make_video(10, 320, 320, seed=4, n_obj=3)
    u8 = frames.round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()
    ref, got = Recorder(), Recorder()
    seq = UnicornMOTTracker(eng, (320, 320), conf=0.01, nms=0.7, assoc="byte", tracker=ref)
    for t in range(10):
        seq.step_tensor(u8[t:t + 1], img_info=(320, 320))
    pipe = UnicornMOTTracker(eng, (320, 320), conf=0.01, nms=0.7, assoc="byte", tracker=got, use_graph=True, depth=3)
    sub = 0
    for t in range(10):
        while sub < 10 and sub - t < 3:
            pipe.submit(u8[sub:sub + 1].pin_memory())
            sub += 1
        pipe.collect((320, 320))
    assert all(c.graph is not None for c in pipe._ctxs)
    assert len(ref.rows) == len(got.rows) == 10 and sum(r.shape[0] for r in ref.rows) > 10
    for t, (r, g) in enumerate(zip(ref.rows, got.rows)):
        assert r.shape == g.shape and torch.equal(r, g), f"frame {t}"
    # n_seq = 2, three steps in flight: the second sequence is the first one's frames in reverse order
    from unicorn_b200.mot import UnicornMOTBatch
    steps = torch.stack([u8, u8.flip(0)], 1)  # [10, 2, H, W, 3]
    seqs, pipes = [Recorder(), Recorder()], [Recorder(), Recorder()]
    seq2 = UnicornMOTBatch(eng, (320, 320), 2, conf=0.01, nms=0.7, assoc="byte")
    pipe2 = UnicornMOTBatch(eng, (320, 320), 2, conf=0.01, nms=0.7, assoc="byte", use_graph=True, depth=3)
    for i in range(2):
        seq2.start(i, seqs[i])
        pipe2.start(i, pipes[i])
    for t in range(10):
        seq2.step_tensor(steps[t], img_infos=[(320, 320)] * 2)
    sub = 0
    for t in range(10):
        while sub < 10 and sub - t < 3:
            pipe2.submit(steps[sub].pin_memory())
            sub += 1
        pipe2.collect([(320, 320)] * 2)
    assert all(c.graph is not None for c in pipe2._ctxs)
    for i in range(2):
        assert len(seqs[i].rows) == len(pipes[i].rows) == 10
        for t, (r, g) in enumerate(zip(seqs[i].rows, pipes[i].rows)):
            assert r.shape == g.shape and torch.equal(r, g), f"sequence {i} frame {t}"
    assert all(torch.equal(r, g) for r, g in zip(ref.rows, seqs[0].rows))


def test_byte_tracker_matches_reference_logic():
    """30 frames of seeded detections through BYTETracker.update vs the reference's own update() flow
    (tests/golden/byte_tracker.npz: reference STrack/Kalman/association code with lap/cython_bbox emulated)."""
    import types
    from unicorn_b200.synthetic import make_detections
    from unicorn_b200.tracker import BYTETracker
    from unicorn_b200.tracker.byte_tracker import STrack
    g = np.load(os.path.join(ROOT, "tests", "golden", "byte_tracker.npz"))
    args = types.SimpleNamespace(track_thresh=0.6, track_buffer=30, match_thresh=0.9, mot20=False)
    STrack._count = 0
    trk = BYTETracker(args)
    frames = make_detections(int(g["n_frames"]), int(g["n_obj"]), int(g["seed"]))
    for i, (boxes, _) in enumerate(frames):
        out = trk.update(boxes.numpy().copy(), (800, 1280), (800, 1280))
        rows = np.array([[t.track_id, *t.tlwh, t.score] for t in out]).reshape(-1, 6)
        rows = rows[np.argsort(rows[:, 0])] if len(rows) else rows
        ref = g[f"f{i}"]
        assert rows.shape == ref.shape, (i, rows[:, 0], ref[:, 0])
        assert np.array_equal(rows[:, 0], ref[:, 0]), (i, rows[:, 0], ref[:, 0])   # bit-matching track ids
        assert np.allclose(rows[:, 1:], ref[:, 1:], rtol=1e-4, atol=1e-2), (i, np.abs(rows - ref).max())
    assert STrack._count == int(g["total_ids"])

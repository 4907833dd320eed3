"""Several MOTS sequences in one batched frame: the batched encode (uc_mots_encode_batched) against one-image encodes of each image, and
UnicornMOTSBatch against one UnicornMOTSTracker per sequence (frame id, ids, category, sizes and RLE strings of every frame)."""
import pytest
import torch

from test_mots_encode_gpu import SIZES, THR, blob_masks, order_and_emit, ratio

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ encoder
def single(masks, order, emit, r, h, w):
    """One-image encode (uc_mots_encode): (chars bytes, offsets list)."""
    from unicorn_b200 import ops
    k = order.numel()
    ws = ops.mots_encode_workspace(k, h, w, "cuda")
    chars, offs = torch.zeros(1 << 22, dtype=torch.uint8, device="cuda"), torch.zeros(k + 1, dtype=torch.int64, device="cuda")
    ops.mots_encode(masks, order.cuda(), torch.tensor(emit, dtype=torch.uint8, device="cuda"), THR, r, h, w, ws, chars, offs)
    o = offs.tolist()
    return bytes(chars[:o[-1]].cpu().numpy()), o


def batched(masks, orders, emits, rs, hs, ws_, cap=1 << 22):
    """One batched encode over the images: per image (chars bytes, offsets relative to the image's first string)."""
    from unicorn_b200 import ops
    ks = [o.numel() for o in orders]
    K = sum(ks)
    ws = ops.mots_encode_workspace(K, max(hs), max(ws_), "cuda")
    chars, offs = torch.zeros(cap, dtype=torch.uint8, device="cuda"), torch.zeros(K + 1, dtype=torch.int64, device="cuda")
    order = torch.cat(orders).to(torch.int32).cuda()
    emit = torch.tensor([e for em in emits for e in em], dtype=torch.uint8, device="cuda")
    ops.mots_encode(masks, order, emit, THR, rs, hs, ws_, ws, chars, offs, k=ks)
    o, out, j = offs.tolist(), [], 0
    for k in ks:
        out.append((bytes(chars[o[j]:o[j + k]].cpu().numpy()), [v - o[j] for v in o[j:j + k + 1]]))
        j += k
    return out


@pytest.fixture(scope="module")
def four():
    """Four different [64, 800, 1280] mask blocks, one per image."""
    return torch.stack([blob_masks(64, b) for b in range(4)])


def test_batched_encode_equals_one_image_encodes(four):
    """The four sizes of test_mots_encode_gpu (r = 1, 401-row masks included) with k = 0, 1, 20 and 64, a mix of emit and the special
    rows, in one encode; each image byte-identical to its own uc_mots_encode."""
    ks = [0, 1, 20, 64]
    orders, emits = zip(*[order_and_emit(k, 64, 10 + b) for b, k in enumerate(ks)])
    hs, ws = [h for h, _ in SIZES], [w for _, w in SIZES]
    rs = [ratio(h, w) for h, w in SIZES]
    got = batched(four, orders, emits, rs, hs, ws)
    assert got[0] == (b"", [0])  # k = 0: no string (the one-image call needs a non-empty order)
    for b in range(1, 4):
        want = single(four[b], orders[b], emits[b], rs[b], hs[b], ws[b])
        assert got[b] == want, f"image {b} ({SIZES[b]}, k = {ks[b]})"
    assert len(got[3][0]) > 0 and not all(emits[3])


def test_identical_images_encode_identically(four):
    """Overlap removal stays within an image: two images with the same masks and order encode as one does alone."""
    order, emit = order_and_emit(20, 64, 7)
    h, w = 480, 640
    masks = torch.stack([four[0], four[0]])
    got = batched(masks, [order, order], [emit, emit], [ratio(h, w)] * 2, [h, h], [w, w])
    assert got[0] == got[1] == single(four[0], order, emit, ratio(h, w), h, w)


def test_encoder_batch_grows_its_buffer_once():
    from unicorn_b200 import _lib
    from unicorn_b200.mots import MaskEncoder
    h, w = 720, 1280  # r = 1: the checkerboards stay checkerboards, about one char per pixel
    cb = ((torch.arange(800)[:, None] + torch.arange(1280)[None, :]) % 2).float()
    masks = torch.stack([torch.stack([cb, 1 - cb]), torch.stack([1 - cb, cb])]).cuda()
    frames = [([0, 1], [True, True], 1.0, h, w), None, ([1], [True], 1.0, h, w)]
    masks3 = torch.cat([masks, masks[:1]])
    small, large = MaskEncoder(6, "cuda", capacity=64), MaskEncoder(6, "cuda", capacity=1 << 22)
    l0 = _lib.LAUNCHES
    got = small.batch(masks3, THR, frames)
    assert _lib.LAUNCHES - l0 == 6, "one encode, one more after the buffer grew"
    assert got == large.batch(masks3, THR, frames)
    assert got[1] == [] and len(got[0]) == 2 and len(got[2]) == 1 and small.d_chars.numel() >= sum(len(s) for f in got for s in f)
    assert got[0] == large(masks3[0], [0, 1], [True, True], THR, 1.0, h, w) and got[2] == large(masks3[2], [1], [True], THR, 1.0, h, w)


def test_captured_batched_encode_equals_eager(four):
    from unicorn_b200 import ops
    ks, sizes = [20, 5, 0], [(402, 640), (1080, 1920), (480, 640)]
    orders, emits = zip(*[order_and_emit(k, 64, 20 + b) for b, k in enumerate(ks)])
    hs, ws_ = [h for h, _ in sizes], [w for _, w in sizes]
    rs = [ratio(h, w) for h, w in sizes]
    ws = ops.mots_encode_workspace(sum(ks), 1080, 1920, "cuda")
    order = torch.cat(orders).to(torch.int32).cuda()
    emit = torch.tensor([e for em in emits for e in em], dtype=torch.uint8, device="cuda")
    masks = four[:3]
    eager_c, eager_o = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda"), torch.zeros(26, dtype=torch.int64, device="cuda")
    ops.mots_encode(masks, order, emit, THR, rs, hs, ws_, ws, eager_c, eager_o, k=ks)
    chars, offs = torch.zeros_like(eager_c), torch.zeros_like(eager_o)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.mots_encode(masks, order, emit, THR, rs, hs, ws_, ws, chars, offs, k=ks)
    g.replay()
    torch.cuda.synchronize()
    n = int(eager_o[-1])
    assert n > 0 and torch.equal(offs, eager_o) and torch.equal(chars[:n], eager_c[:n])


# ------------------------------------------------------------------------------------------------ driver
SIZE = (320, 320)
KW = dict(conf=0.01, nms=0.7, score_thr=0.02, max_dets=16, min_box_area=300)  # the lowered gates of test_mots_encode_gpu
ORIG = [(201, 201), (480, 640), (320, 320), (402, 640)]  # original (h, w) of sequences 0..3


def qd_tracker():
    from unicorn_b200.tracker import QuasiDenseEmbedTracker
    return QuasiDenseEmbedTracker(init_score_thr=0.05, obj_score_thr=0.03)


@pytest.fixture(scope="module")
def tiny():
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.weights import make_state_dict
    name = "unicorn_track_tiny_mask"
    eng = UnicornEngine(make_state_dict(name, 0), name)
    return eng, [make_video(6, *SIZE, seed=1 + s, n_obj=3)[0] for s in range(4)]


def reference(eng, frames, size, kw=KW, input_size=SIZE):
    """One UnicornMOTSTracker fed `frames` (each [1,...]) of original size `size`: its write_results_mots() tuples."""
    from unicorn_b200.mots import UnicornMOTSTracker
    trk = UnicornMOTSTracker(eng, input_size, tracker=qd_tracker(), **kw)
    return [trk.step_tensor(f, *size) for f in frames]


def run_batch(eng, n_seq, steps, use_graph, pipelined, kw=KW):
    """steps: per step {"start": [slots started before it], "frames": n_seq frames [3,H,W] or None (idle), "sizes": n_seq (h, w)}."""
    from unicorn_b200.mots import UnicornMOTSBatch
    mb = UnicornMOTSBatch(eng, SIZE, n_seq, use_graph=use_graph, **kw)
    filler = torch.zeros(3, *SIZE)
    results, graphs = [], []

    def submit(t):
        for i in steps[t].get("start", []):
            if use_graph and t >= 4:
                graphs.append([c.graph for c in mb._ctxs])
            mb.start(i, qd_tracker())
        fr = steps[t]["frames"]
        mb.submit(torch.stack([f if f is not None else filler for f in fr]), steps[t]["sizes"], active=[f is not None for f in fr])

    if pipelined:
        submit(0)
        for t in range(len(steps)):
            if t + 1 < len(steps):
                submit(t + 1)
            results.append(mb.collect())
    else:
        for t in range(len(steps)):
            submit(t)
            results.append(mb.collect())
    if use_graph:
        assert len(mb._graphs) == 2
        for gs in graphs:  # start() after the captures did not re-capture
            assert all(a is b for a, b in zip(gs, [c.graph for c in mb._ctxs]))
    return mb, results


def encoded(results):
    return sum(len(r[5]) for step in results for r in (step if isinstance(step, list) else [step]) if r is not None)


@pytest.mark.parametrize("use_graph,pipelined", [(False, False), (True, False), (True, True)], ids=["eager", "graph", "pipelined"])
def test_batch_matches_separate_trackers(tiny, use_graph, pipelined):
    eng, videos = tiny
    T = 5
    refs = [reference(eng, [v[t:t + 1] for t in range(T)], ORIG[s]) for s, v in enumerate(videos[:3])]
    steps = [{"start": [0, 1, 2] if t == 0 else [], "frames": [v[t] for v in videos[:3]], "sizes": ORIG[:3]} for t in range(T)]
    _, got = run_batch(eng, 3, steps, use_graph, pipelined)
    assert encoded(refs) > 0, "no instance was encoded: a vacuous test"
    for t in range(T):
        for s in range(3):
            assert got[t][s] == refs[s][t], f"step {t} sequence {s}"


def test_single_sequence_equals_tracker(tiny):
    eng, videos = tiny
    T = 5
    ref = reference(eng, [videos[3][t:t + 1] for t in range(T)], ORIG[3])
    steps = [{"start": [0] if t == 0 else [], "frames": [videos[3][t]], "sizes": ORIG[3:]} for t in range(T)]
    _, got = run_batch(eng, 1, steps, use_graph=True, pipelined=True)
    assert encoded(ref) > 0
    assert [g[0] for g in got] == ref


def test_idle_unstarted_and_restarted_slots(tiny):
    """Slot 0 runs throughout; slot 1 sits out step 2 (against a tracker that skipped that frame); slot 2 is not started before step 2,
    then runs video C, and is restarted with video D at step 4 (against fresh trackers)."""
    eng, (va, vb, vc, vd) = tiny
    T = 6
    steps = []
    for t in range(T):
        c = None if t < 2 else vc[t - 2] if t < 4 else vd[t - 4]
        steps.append({"start": [0, 1] if t == 0 else [2] if t in (2, 4) else [], "frames": [va[t], None if t == 2 else vb[t], c],
                      "sizes": [ORIG[0], ORIG[1], ORIG[2] if t < 4 else ORIG[3]]})
    ref0 = reference(eng, [va[t:t + 1] for t in range(T)], ORIG[0])
    ref1 = reference(eng, [vb[t:t + 1] for t in range(T) if t != 2], ORIG[1])
    ref2a, ref2b = reference(eng, [vc[t:t + 1] for t in range(2)], ORIG[2]), reference(eng, [vd[t:t + 1] for t in range(2)], ORIG[3])
    _, got = run_batch(eng, 3, steps, use_graph=True, pipelined=True)
    assert encoded(ref0) + encoded(ref1) > 0
    k1 = 0
    for t in range(T):
        assert got[t][0] == ref0[t], f"step {t} slot 0"
        if t == 2:
            assert got[t][1] is None
        else:
            assert got[t][1] == ref1[k1], f"step {t} slot 1"
            k1 += 1
        want2 = None if t < 2 else ref2a[t - 2] if t < 4 else ref2b[t - 4]
        assert got[t][2] == want2, f"step {t} slot 2"


def test_launches_per_step_do_not_depend_on_n_seq(tiny):
    """The batched frame and the batched encode launch as many kernels for three sequences as for one (each sequence's tracker
    launches its own matching kernels on the host half)."""
    from unicorn_b200 import _lib
    from unicorn_b200.mots import UnicornMOTSBatch
    eng, (va, _, _, _) = tiny
    frame_launches, encode_launches = [], {1: [], 3: []}
    for n in (1, 3):
        mb = UnicornMOTSBatch(eng, SIZE, n, **KW)
        for i in range(n):
            mb.start(i, qd_tracker())
        batch = mb._enc.batch

        def counted(*a, batch=batch, n=n):
            l0 = _lib.LAUNCHES
            out = batch(*a)
            encode_launches[n].append(_lib.LAUNCHES - l0)
            return out
        mb._enc.batch = counted
        for t in range(3):  # the same frames in every slot: the same instances to encode
            res = mb.step_tensor(torch.stack([va[t]] * n), [ORIG[0]] * n)
            assert all(r == res[0] for r in res)
        frame_launches.append(mb.launches_per_frame)
    assert frame_launches[0] == frame_launches[1] > 0, frame_launches
    assert encode_launches[1] == encode_launches[3] and 3 in encode_launches[1], encode_launches


def test_validation_and_failed_copy_leave_state_unchanged(tiny, monkeypatch):
    from unicorn_b200.frames import FrameSlot
    from unicorn_b200.mots import UnicornMOTSBatch
    eng, (va, vb, vc, _) = tiny
    mb = UnicornMOTSBatch(eng, SIZE, 3, **KW)
    for i in range(3):
        mb.start(i, qd_tracker())
    mb.step_tensor(torch.stack([va[0], vb[0], vc[0]]), ORIG[:3])
    torch.cuda.synchronize()

    def state():
        nxt = mb._ctxs[mb._ring.submitted % 2]
        return (list(mb.frame_ids), mb._ring.submitted, mb.has_prev.clone().tolist(), mb.prev_feat.float().sum().item(), list(nxt.mask),
                list(nxt.img_hw), nxt.u8, nxt.graph)
    before = state()
    good = torch.stack([va[1], vb[1], vc[1]])
    for kw in (dict(frames=good[:2]), dict(frames=good.double()), dict(frames=good, active=[1, 1]), dict(img_sizes=ORIG[:2]),
               dict(img_sizes=[(201, 201), (0, 640), (320, 320)]), dict(img_sizes=None), dict(img_sizes=[(1, 2, 3)] * 3)):
        args = dict(dict(frames=good, img_sizes=ORIG[:3]), **kw)
        with pytest.raises(ValueError):
            mb.submit(**args)
    torch.cuda.synchronize()
    assert state() == before

    def fail(self, frames):
        raise RuntimeError("copy failed")
    with monkeypatch.context() as m:
        m.setattr(FrameSlot, "stage", fail)
        with pytest.raises(RuntimeError):
            mb.submit(good, ORIG[1:4], active=[True, False, True])
    assert state() == before
    res = mb.step_tensor(good, ORIG[:3])
    assert all(r is not None and r[0] == 2 for r in res) and mb.frame_ids == [2, 2, 2]


# ------------------------------------------------------------------------------------------------ full size
def test_full_size_matches_separate_trackers():
    """unicorn_track_large_mot_challenge_mask at 800x1280, two sequences from 1080x1920 and 480x640 frames."""
    from unicorn_b200 import ops
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.weights import make_state_dict
    name, size, T = "unicorn_track_large_mot_challenge_mask", (800, 1280), 3
    eng = UnicornEngine(make_state_dict(name, 0), name)
    origs = [(1080, 1920), (480, 640)]
    seqs = []
    for s, (h, w) in enumerate(origs):
        raw = make_video(T, h, w, seed=5 + s, n_obj=4)[0].round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous().cuda()
        seqs.append(torch.cat([ops.letterbox_u8(raw[t], size, swap_rb=False)[0] for t in range(T)]))
    from unicorn_b200.tracker import QuasiDenseEmbedTracker
    kw = dict(conf=0.01, nms=0.7, score_thr=0.0, max_dets=64, min_box_area=0)
    mk = lambda: QuasiDenseEmbedTracker(init_score_thr=0.0, obj_score_thr=0.0)  # noqa: E731
    from unicorn_b200.mots import UnicornMOTSBatch, UnicornMOTSTracker
    refs = []
    for s in range(2):
        trk = UnicornMOTSTracker(eng, size, tracker=mk(), use_graph=True, **kw)
        refs.append([trk.step_tensor(seqs[s][t:t + 1], *origs[s]) for t in range(T)])
    mb = UnicornMOTSBatch(eng, size, 2, use_graph=True, **kw)
    for s in range(2):
        mb.start(s, mk())
    got = [mb.step_tensor(torch.stack([seqs[0][t], seqs[1][t]]), origs) for t in range(T)]
    assert encoded(refs) > 0, "no instance was encoded"
    for t in range(T):
        for s in range(2):
            assert got[t][s] == refs[s][t], f"step {t} sequence {s}"

"""BDD100K MOTS bitmasks on the H100 (BDDBitmasks / uc_bdd_bitmask_batched) byte for byte against the numpy restatement of qdtrack's
mask_prepare + mask_merge (oracle/bdd_bitmask_oracle.py) and the unmodified reference's PNGs (tests/golden/bdd_bitmask.npz):
overlaps, ties under an explicit order, the channel arithmetic, empty / full / leading-foreground masks and runs across columns,
frames without tracks and of mixed sizes in one batch, 64 full-size frames, malformed strings, graph capture, and the tracker's own
track_result dicts end to end."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bdd_bitmask_oracle as bo  # noqa: E402
from test_bdd_bitmask import check_synthetic, load_golden, synthetic_dicts, tiny_dicts  # noqa: E402

GUARD = 0xAB  # what the tests' output buffers hold before a call: every frame byte must be written, nothing else


@pytest.fixture(scope="module")
def golden():
    return load_golden()


@pytest.fixture(scope="module")
def painter():
    from unicorn_b200.bdd import BDDBitmasks
    return BDDBitmasks("cuda")


def host(views):
    return [v.cpu().numpy() for v in views]


def instance(tid, label, score, mask):
    from unicorn_b200.results import rle_dict, rle_encode
    h, w = mask.shape
    return np.int64(tid), dict(bbox=np.array([0, 0, 1, 1, score], dtype=np.float32), label=np.float32(label), segm=rle_dict(rle_encode(mask), h, w))


def random_frame(rng, h, w, k, ids=None):
    """k instances on an h x w frame: ellipses and rectangles (some full height), distinct scores, labels 0..7."""
    yy, xx = np.mgrid[:h, :w]
    scores = rng.permutation(100000)[:k].astype(np.float32) / 100000
    d = {}
    for n in range(k):
        cy, cx, ry, rx = rng.integers(0, h), rng.integers(0, w), rng.integers(1, max(2, h // 3)), rng.integers(1, max(2, w // 3))
        m = ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 <= 1.0 if n % 3 else (abs(xx - cx) <= rx // 4) & (yy >= cy // 2)
        tid = ids[n] if ids is not None else int(rng.integers(0, 1 << 17))
        t, v = instance(tid, n % 8, scores[n], m)
        d[t] = v
    return d


def launch(dicts, sizes, ranks=None, strings=None, gap=64):
    """uc_bdd_bitmask_batched through the launcher, the frames `gap` bytes apart in a buffer of GUARD bytes: (bitmasks, status,
    whether every byte outside the frames kept its value).  ranks / strings: per frame, overriding what the painter would pass."""
    from unicorn_b200 import post_ops
    from unicorn_b200.bdd import _frame
    per = [_frame(d, h, w, f) for f, (d, (h, w)) in enumerate(zip(dicts, sizes))]
    s = [x for f, p in enumerate(per) for x in (strings[f] if strings and strings[f] is not None else p[0])]
    colors = np.concatenate([p[1] for p in per] + [np.zeros(1, np.uint32)]).view(np.int32)
    rk = np.concatenate([np.asarray(ranks[f] if ranks and ranks[f] is not None else p[2], dtype=np.int32) for f, p in enumerate(per)]
                        + [np.zeros(1, np.int32)])
    k = [len(p[0]) for p in per]
    hs, ws = [h for h, _ in sizes], [w for _, w in sizes]
    chars = b"".join(s)
    offsets = np.concatenate([[0], np.cumsum([len(x) for x in s])]).astype(np.int64)
    out_off = np.concatenate([[0], np.cumsum([4 * h * w + gap for h, w in sizes])]).astype(np.int64)
    out = torch.full((int(out_off[-1]) + 4096,), GUARD, dtype=torch.uint8, device="cuda")
    ws_buf = torch.empty(post_ops.bdd_bitmask_workspace_bytes(k, hs, ws, len(chars)), dtype=torch.uint8, device="cuda")
    status = torch.full((len(k),), -1, dtype=torch.int32, device="cuda")
    dev = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a)).to(dt).cuda()  # noqa: E731
    post_ops.bdd_bitmask(dev(np.frombuffer(chars + b"\0", dtype=np.uint8), torch.uint8), len(chars), dev(offsets, torch.int64),
                         dev(colors, torch.int32), dev(rk, torch.int32), k, hs, ws, out, out_off[:-1].tolist(), ws_buf, status)
    torch.cuda.synchronize()
    o = out.cpu().numpy()
    frames = [o[out_off[f]:out_off[f] + 4 * h * w].reshape(h, w, 4).copy() for f, (h, w) in enumerate(sizes)]
    for f, (h, w) in enumerate(sizes):
        o[out_off[f]:out_off[f] + 4 * h * w] = GUARD
    return frames, status.tolist(), bool((o == GUARD).all())


def painted_in_order(d, h, w, order):
    """mask_merge with the paint order given instead of np.argsort(scores)."""
    _, colors, masks = bo.mask_prepare(d)
    bm = np.zeros((h, w, 4), dtype=np.uint8)
    for idx in order:
        for i in range(4):
            bm[..., i] = bm[..., i] * (1 - masks[idx]) + masks[idx] * colors[idx][i]
    return bm


# ------------------------------------------------------------------------------------------------ against the reference's PNGs
def test_golden_frames(painter, golden):
    dicts, (h, w) = tiny_dicts()
    for f, bm in enumerate(host(painter.paint(dicts, [(h, w)] * len(dicts)))):
        assert np.array_equal(bm, golden["tiny_bitmask"][f]), f
    syn = synthetic_dicts(golden)  # 720 x 1280 twice, 1 x 1, 7 x 13, 7 x 13 without tracks: mixed sizes and K = 0 in one batch
    batch = host(painter.paint([d for d, _ in syn], [hw for _, hw in syn]))
    for c, bm in enumerate(batch):
        check_synthetic(golden, c, bm)
    for c, (d, hw) in enumerate(syn):  # B = 1 equals B = n
        assert np.array_equal(host(painter.paint([d], [hw]))[0], batch[c]), c
    frames, status, clean = launch([d for d, _ in syn], [hw for _, hw in syn])
    assert status == [0] * len(syn) and clean
    assert all(np.array_equal(a, b) for a, b in zip(frames, batch))


def test_host_readback_equals_the_device_views(painter, golden):
    syn = synthetic_dicts(golden)
    dev = host(painter.paint([d for d, _ in syn], [hw for _, hw in syn]))
    hst = painter.paint([d for d, _ in syn], [hw for _, hw in syn], host=True)
    assert all(isinstance(a, np.ndarray) and np.array_equal(a, b) for a, b in zip(hst, dev))


# ------------------------------------------------------------------------------------------------ against the oracle
def test_overlaps_ids_labels_and_mask_shapes(painter):
    rng = np.random.default_rng(5)
    h, w = 720, 1280
    ids = [0, 255, 256, 65535, 65536, 1, 511, 131071, 70000, 3] * 3
    frames = [random_frame(rng, h, w, 30, ids)]
    yy, xx = np.mgrid[:h, :w]
    special = [instance(1, 0, 0.1, np.zeros((h, w), bool)), instance(2, 1, 0.05, np.ones((h, w), bool)),  # empty, full
               instance(3, 2, 0.5, (yy < 10) & (xx < 3)),  # first pixel foreground
               instance(4, 3, 0.6, (xx == 5) & (yy > 700) | (xx == 6) & (yy < 20)),  # one run from the bottom of a column into the next
               instance(5, 4, 0.7, (xx >= 1270) & (yy >= 710)),  # ends at the last pixel
               instance(65536, 7, 0.9, (yy % 2 == 0) & (xx % 3 == 0))]  # single-pixel runs
    frames.append(dict(special))
    frames.append({})
    small = [(1, 1), (7, 13), (33, 65)]
    for hh, ww in small:
        frames.append(random_frame(rng, hh, ww, 9))
    sizes = [(h, w), (h, w), (h, w)] + small
    got = host(painter.paint(frames, sizes))
    for f, (d, (hh, ww)) in enumerate(zip(frames, sizes)):
        assert np.array_equal(got[f], bo.bdd_bitmask(d, hh, ww)), f
    colors = {tuple(int(c) for c in v) for v in got[1].reshape(-1, 4)}
    assert {(8, 0, 0, 0), (4, 0, 0, 4), (3, 0, 0, 3), (2, 0, 0, 2)} <= colors  # id 65536 wraps B to 0; the band, the corner, the full mask
    assert len({tuple(v) for v in got[0].reshape(-1, 4)}) >= 10


def test_ties_follow_the_given_order(painter):
    rng = np.random.default_rng(9)
    h, w = 48, 40
    yy, xx = np.mgrid[:h, :w]
    d = dict(instance(10 + n, n, 0.5, ((yy - 20 - n) / 18) ** 2 + ((xx - 18 - n) / 15) ** 2 <= 1) for n in range(6))  # all tied, all overlap
    d.update([instance(99, 7, 0.25, xx < 30), instance(98, 6, 0.75, yy < 8)])
    assert np.array_equal(host(painter.paint([d], [(h, w)]))[0], bo.bdd_bitmask(d, h, w))  # np.argsort's own tie order
    for order in (np.arange(8), np.arange(8)[::-1], rng.permutation(8)):
        ranks = np.empty(8, dtype=np.int32)
        ranks[order] = np.arange(8)
        frames, status, clean = launch([d], [(h, w)], ranks=[ranks])
        assert status == [0] and clean
        assert np.array_equal(frames[0], painted_in_order(d, h, w, order)), order


def test_64_full_size_frames(painter):
    rng = np.random.default_rng(64)
    frames = [random_frame(rng, 720, 1280, int(rng.integers(0, 25))) for _ in range(64)]
    frames[17] = {}
    got = host(painter.paint(frames, [(720, 1280)] * 64))
    for f in (0, 17, 40, 63):
        assert np.array_equal(got[f], bo.bdd_bitmask(frames[f], 720, 1280)), f
    for f in range(64):
        assert np.array_equal(got[f], host(painter.paint([frames[f]], [(720, 1280)]))[0]), f
    assert not got[17].any()


def test_malformed_strings(painter):
    """Each malformed string is reported in its frame's status and paints nothing; the other frames are as without it."""
    from unicorn_b200 import post_ops
    from unicorn_b200.results import rle_encode
    rng = np.random.default_rng(3)
    h, w = 24, 20
    good = rle_encode(rng.random((h, w)) < 0.3).encode()
    cases = [
        (b"~" + good[1:], post_ops.BDD_BAD_CHARS),  # a char past 'o'
        (b"/" + good[1:], post_ops.BDD_BAD_CHARS),  # a char before '0'
        (good + b"h", post_ops.BDD_BAD_CHARS),  # ends inside a count (continuation bit)
        (b"0" + b"h" * 7 + b"0", post_ops.BDD_BAD_CHARS),  # an 8-char count
        (b"", post_ops.BDD_BAD_RUNS),  # no runs
        (rle_encode(np.zeros((h, w - 1), bool)).encode(), post_ops.BDD_BAD_RUNS),  # runs that end early
        (rle_encode(np.zeros((h, w + 1), bool)).encode(), post_ops.BDD_BAD_RUNS),  # runs past the frame
        (rle_encode(np.ones((h, w + 1), bool)).encode(), post_ops.BDD_BAD_RUNS),  # foreground past the frame
        (b"111@", post_ops.BDD_BAD_RUNS),  # 1, 1, 1, then a delta that makes the count negative
    ]
    frames, sizes, strings = [], [], []
    for s, _ in cases:
        d = random_frame(rng, h, w, 4)
        bad_id = list(d)[2]
        frames.append(d)
        sizes.append((h, w))
        strings.append([d[t]["segm"]["counts"] if t != bad_id else s for t in d])
    frames.append(random_frame(rng, h, w, 5))  # a well-formed frame between them
    sizes.append((h, w))
    strings.append(None)
    got, status, clean = launch(frames, sizes, strings=strings)
    assert clean
    assert status == [flag for _, flag in cases] + [0]
    for f, d in enumerate(frames):
        keep = {t: v for t, v in d.items() if f == len(cases) or t != list(d)[2]}
        assert np.array_equal(got[f], bo.bdd_bitmask(keep, h, w)), f
    for f, (s, _) in enumerate(cases):  # the painter raises on the dicts themselves
        bad = {t: dict(v, segm=dict(v["segm"], counts=s)) if t == list(frames[f])[2] else v for t, v in frames[f].items()}
        with pytest.raises(ValueError, match="frame 1: "):
            painter.paint([frames[-1], bad], [(h, w)] * 2)
    assert np.array_equal(host(painter.paint([frames[-1]], [(h, w)]))[0], bo.bdd_bitmask(frames[-1], h, w))  # usable afterwards


def test_graph_capture():
    from unicorn_b200 import post_ops
    from unicorn_b200.bdd import _frame
    rng = np.random.default_rng(1)
    dicts = [random_frame(rng, 96, 128, 12), {}, random_frame(rng, 50, 30, 4)]
    sizes = [(96, 128), (96, 128), (50, 30)]
    per = [_frame(d, h, w, f) for f, (d, (h, w)) in enumerate(zip(dicts, sizes))]
    s = [x for p in per for x in p[0]]
    k, hs, ws = [len(p[0]) for p in per], [h for h, _ in sizes], [w for _, w in sizes]
    chars = torch.tensor(list(b"".join(s)), dtype=torch.uint8, device="cuda")
    offsets = torch.tensor(np.concatenate([[0], np.cumsum([len(x) for x in s])]), dtype=torch.int64, device="cuda")
    colors = torch.from_numpy(np.concatenate([p[1] for p in per]).view(np.int32)).cuda()
    ranks = torch.from_numpy(np.concatenate([p[2] for p in per])).cuda()
    out_off = [0, 4 * 96 * 128, 8 * 96 * 128]
    out = torch.zeros(out_off[-1] + 4 * 50 * 30, dtype=torch.uint8, device="cuda")
    wsb = torch.empty(post_ops.bdd_bitmask_workspace_bytes(k, hs, ws, chars.numel()), dtype=torch.uint8, device="cuda")
    status = torch.zeros(3, dtype=torch.int32, device="cuda")
    run = lambda: post_ops.bdd_bitmask(chars, chars.numel(), offsets, colors, ranks, k, hs, ws, out, out_off, wsb, status)  # noqa: E731
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        run()
    torch.cuda.current_stream().wait_stream(stream)
    torch.cuda.synchronize()
    want = out.clone()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        run()
    out.fill_(GUARD)
    status.fill_(-1)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, want) and status.tolist() == [0, 0, 0]
    o = want.cpu().numpy()
    for f, (d, (h, w)) in enumerate(zip(dicts, sizes)):
        assert np.array_equal(o[out_off[f]:out_off[f] + 4 * h * w].reshape(h, w, 4), bo.bdd_bitmask(d, h, w)), f


# ------------------------------------------------------------------------------------------------ end to end
def test_tracker_results_end_to_end(painter, tmp_path):
    """UnicornBDDMOTSBatch on the golden frames, then the bitmasks of its collect() dicts, in one batch and as PNGs."""
    from PIL import Image
    from test_bdd import load_bdd_golden
    from test_bdd_gpu import driver, tracker, video
    from unicorn_b200.bdd import write_seg_track
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.weights import make_state_dict
    g = load_bdd_golden()
    h, w = (int(v) for v in g["orig"])
    trk = driver({True: UnicornEngine(make_state_dict("unicorn_track_tiny_mask", 0), "unicorn_track_tiny_mask")}, True, g)
    trk.start(0, tracker(g, "mots_"))
    frs = video(g)
    results = [trk.step_tensor(frs[f:f + 1], [(h, w)])[0]["track_result"] for f in range(frs.shape[0])]
    assert sum(len(r) for r in results) >= 4
    got = host(painter.paint(results, [(h, w)] * len(results)))
    want = [bo.bdd_bitmask(r, h, w) for r in results]
    assert all(np.array_equal(a, b) for a, b in zip(got, want))
    assert any(b.any() for b in want)
    names = [f"seq/seq-{f:07d}.jpg" for f in range(len(results))]
    paths = write_seg_track(results, names, str(tmp_path), [(h, w)] * len(results), painter=painter, batch=3)
    for p, b in zip(paths, want):
        assert np.array_equal(np.asarray(Image.open(p)), b), p

"""BDD100K MOTS bitmasks (qdtrack's seg_track format) without a GPU: the numpy oracle (oracle/bdd_bitmask_oracle.py) against the
unmodified mask_prepare + mask_merge (tests/golden/bdd_bitmask.npz, written by tests/golden/make_golden_bdd_bitmask.py), the PNG
writer's files and paths, the argument validation of uc_bdd_bitmask_batched (fake pointers, rejected before any CUDA call) and the
painter's frame-size check."""
import ctypes
import hashlib
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import bdd_bitmask_oracle as bo  # noqa: E402
from make_golden_bdd_bitmask import SMALL, rasterise, synthetic_cases, tiny_frames  # noqa: E402


def load_golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "bdd_bitmask.npz"))


def tiny_dicts():
    """The 8 MOTS frames of bdd_tiny_320.npz as track_result dicts with COCO RLE segms, and their size."""
    from unicorn_b200.results import rle_dict, rle_encode
    g = np.load(os.path.join(ROOT, "tests", "golden", "bdd_tiny_320.npz"))
    h, w = (int(v) for v in g["orig"])
    return [{tid: dict(bbox=bbox, label=label, segm=rle_dict(rle_encode(m), h, w)) for tid, bbox, label, m in fr} for fr in tiny_frames(g)], (h, w)


def synthetic_dicts(g):
    """The synthetic cases as (track_result dict, (h, w)) from the fixture's strings."""
    out, j = [], 0
    for (h, w), k in zip(g["syn_hw"], g["syn_k"]):
        h, w = int(h), int(w)
        d = {}
        for n in range(j, j + int(k)):
            bbox = np.array([0, 0, 0, 0, g["syn_score"][n]], dtype=np.float32)
            d[np.int64(g["syn_id"][n])] = dict(bbox=bbox, label=g["syn_label"][n], segm={"size": [h, w], "counts": str(g["syn_rle"][n]).encode()})
        out.append((d, (h, w)))
        j += int(k)
    return out


def check_synthetic(g, c, bitmask):
    """Bitmask of synthetic case c against the fixture: whole for small frames, by digest for the others."""
    h, w = (int(v) for v in g["syn_hw"][c])
    assert bitmask.shape == (h, w, 4) and bitmask.dtype == np.uint8
    if h * w <= SMALL:
        assert np.array_equal(bitmask, g[f"syn_bitmask_{c}"]), c
    assert hashlib.sha256(np.ascontiguousarray(bitmask).tobytes()).hexdigest() == str(g["syn_digest"][c]), c


@pytest.fixture(scope="module")
def golden():
    return load_golden()


def test_fixture_strings_are_the_stored_parameters(golden):
    from unicorn_b200.results import rle_encode
    g, j = golden, 0
    for c, (h, w, insts) in enumerate(synthetic_cases()):
        assert (int(g["syn_hw"][c][0]), int(g["syn_hw"][c][1])) == (h, w) and int(g["syn_k"][c]) == len(insts)
        for tid, label, score, kind, p in insts:
            assert (g["syn_id"][j], g["syn_label"][j], g["syn_score"][j], g["syn_kind"][j]) == (tid, np.float32(label), np.float32(score), kind)
            assert str(g["syn_rle"][j]) == rle_encode(rasterise(kind, p, h, w))
            j += 1


def test_oracle_equals_the_reference_on_the_tiny_frames(golden):
    dicts, (h, w) = tiny_dicts()
    assert len(dicts) == golden["tiny_bitmask"].shape[0] == 8 and sum(len(d) for d in dicts) > 4
    for f, d in enumerate(dicts):
        assert np.array_equal(bo.bdd_bitmask(d, h, w), golden["tiny_bitmask"][f]), f


def test_oracle_equals_the_reference_on_the_synthetic_frames(golden):
    for c, (d, (h, w)) in enumerate(synthetic_dicts(golden)):
        check_synthetic(golden, c, bo.bdd_bitmask(d, h, w))


def test_channel_arithmetic(golden):
    """R = label + 1 truncated, G = 0, B = (id >> 8) mod 256, A = id & 255, all four from the winner; nothing else is painted."""
    d, (h, w) = synthetic_dicts(golden)[3]
    bm = golden["syn_bitmask_3"]
    colors = {tuple(v) for v in bm.reshape(-1, 4)}
    want = {(int(np.float32(i["label"]) + 1), 0, (int(t) >> 8) % 256, int(t) & 255) for t, i in d.items()}
    assert colors <= want and (3, 0, 1, 0) in colors  # label 2.5, id 256
    assert (2, 0, 255, 255) in colors and (1, 0, 0, 0) in colors  # label 1, id 65535; label 0, id 65536: B wraps to 0
    assert np.array_equal(golden["syn_bitmask_2"].reshape(4), [4, 0, 0, 6])  # 1 x 1: the higher of the two full masks
    assert not golden["syn_bitmask_4"].any()  # no tracks: all zeros


def test_painter_colours_and_ranks_are_mask_prepare_and_argsort(golden):
    """What the painter packs on the host: each instance's colour is the pixel mask_merge paints with it, and the ranks invert
    np.argsort of the scores."""
    from unicorn_b200.bdd import _frame
    dicts, (h, w) = tiny_dicts()
    cases = [(d, (h, w)) for d in dicts] + synthetic_dicts(golden)
    cases.append(({np.int64(t): dict(bbox=np.float32([0, 0, 1, 1, s]), label=np.float32(lab), segm={"size": [1, 1], "counts": b"01"})
                   for t, lab, s in ((0, 0.5, 0.3), (257, 7.99, 0.3), (1 << 40, 3.0, 0.1), (65791, 254.5, 0.2))}, (1, 1)))
    for d, (hh, ww) in cases:
        strings, colors, ranks = _frame(d, hh, ww, 0)
        scores, cols, _ = bo.mask_prepare({t: dict(v, segm={"size": [1, 1], "counts": b"01"}) for t, v in d.items()})
        for c, col, s in zip(colors, cols, strings):
            assert np.array_equal(np.array([c], dtype="<u4").view(np.uint8), bo.mask_merge(([0], [col], [np.ones((1, 1), np.uint8)]), 1, 1)[0, 0])
        assert np.array_equal(np.argsort(ranks), np.argsort(scores)) and sorted(ranks) == list(range(len(d)))
        assert strings == [v["segm"]["counts"] for v in d.values()]


class _OraclePainter:
    """BDDBitmasks' interface on the oracle: what write_seg_track needs without a device."""

    def __init__(self):
        self.calls = []

    def paint(self, track_results, sizes, host=False):
        assert host
        self.calls.append(len(track_results))
        return [bo.bdd_bitmask(d, h, w) for d, (h, w) in zip(track_results, sizes)]


def test_write_seg_track_paths_and_pixels(golden, tmp_path):
    from PIL import Image
    from unicorn_b200.bdd import write_seg_track
    dicts, (h, w) = tiny_dicts()
    syn = synthetic_dicts(golden)[2:]  # the small synthetic frames: mixed sizes in one call
    results = dicts + [d for d, _ in syn]
    sizes = [(h, w)] * len(dicts) + [hw for _, hw in syn]
    names = [f"video-{f // 4}/video-{f // 4}-{f:07d}.jpg" for f in range(len(results))]
    painter = _OraclePainter()
    paths = write_seg_track(results, names, str(tmp_path), sizes, painter=painter, batch=4)
    assert painter.calls == [4, 4, 3]
    want = [golden["tiny_bitmask"][f] for f in range(len(dicts))] + [golden[f"syn_bitmask_{c}"] for c in (2, 3, 4)]
    for name, path, bm in zip(names, paths, want):
        assert path == os.path.join(str(tmp_path), "seg_track", name.replace(".jpg", ".png"))  # seg_track_to_bdd100k + mask_merge
        im = Image.open(path)
        assert im.mode == "RGBA" and im.format == "PNG"
        assert np.array_equal(np.asarray(im), bm), name


def test_painter_rejects_a_segm_of_another_size(golden):
    from unicorn_b200.bdd import BDDBitmasks
    d, (h, w) = synthetic_dicts(golden)[3]
    p = BDDBitmasks("cuda")  # buffers are allocated by the first paint: the checks come first
    with pytest.raises(ValueError, match="segm size"):
        p.paint([d], [(h + 1, w)])
    with pytest.raises(ValueError, match="segm size"):
        p.paint([{}, d], [(4, 4), (w, h)])
    with pytest.raises(ValueError, match="frames"):
        p.paint([{}] * 65, [(1, 1)] * 65)
    with pytest.raises(ValueError, match="frames"):
        p.paint([d], [])
    bad = {np.int64(1): dict(d[next(iter(d))], label=np.float32(255.0))}
    with pytest.raises(ValueError, match="uint8"):
        p.paint([bad], [(h, w)])


# ------------------------------------------------------------------------------------------------ C ABI argument validation
P = ctypes.c_void_p
EINVAL = -1


@pytest.fixture(scope="module")
def lib():
    from unicorn_b200 import _lib
    return _lib.lib()


def bitmask_call(lib, B=2, k=(2, 1), H=(8, 4), W=(8, 4), out_offsets=None, chars=P(0x10000), n_chars=10, offsets=P(0x20000),
                 colors=P(0x30000), ranks=P(0x40000), ws=P(0x50000), ws_bytes=1 << 20, out=P(0x60000), out_bytes=1 << 20,
                 status=P(0x70000)):
    ints = lambda v: (ctypes.c_int * max(len(v), 1))(*v)  # noqa: E731
    if out_offsets is None:
        out_offsets = [sum(4 * H[c] * W[c] for c in range(b)) for b in range(len(H))]
    rc = lib.uc_bdd_bitmask_batched(B, ints(k), ints(H), ints(W), (ctypes.c_long * max(len(out_offsets), 1))(*out_offsets), chars,
                                    ctypes.c_long(n_chars), offsets, colors, ranks, ws, ctypes.c_long(ws_bytes), out, ctypes.c_long(out_bytes),
                                    status, None)
    return rc, lib.uc_last_error()


def rejected(call, *words):
    rc, msg = call
    assert rc == EINVAL, (rc, msg)
    for w in ("uc_bdd_bitmask_batched",) + words:
        assert w.encode() in msg, (w, msg)


def test_bitmask_rejects_bad_frames(lib):
    rejected(bitmask_call(lib, B=0, k=(), H=(), W=()), "B = 0 must be in 1..64")
    rejected(bitmask_call(lib, B=65, k=(0,) * 65, H=(1,) * 65, W=(1,) * 65), "B = 65 must be in 1..64")
    rejected(bitmask_call(lib, H=(0, 4)), "frame 0: bad size")
    rejected(bitmask_call(lib, W=(8, -4)), "frame 1: bad size")
    rejected(bitmask_call(lib, H=(1 << 16, 4), W=(1 << 16, 4)), "frame 0: bad size")
    rejected(bitmask_call(lib, k=(2, -1)), "frame 1: k = -1")
    rejected(bitmask_call(lib, k=(65536, 1)), "frame 0: k = 65536")


def test_bitmask_rejects_bad_pointers_and_alignment(lib):
    for name in ("offsets", "colors", "ranks", "ws", "out", "status"):
        rejected(bitmask_call(lib, **{name: None}), "null pointer")
    rejected(bitmask_call(lib, chars=None), "null pointer")
    rejected(bitmask_call(lib, n_chars=-1), "negative")
    for name, addr in (("colors", 0x30002), ("ranks", 0x40001), ("status", 0x70002), ("out", 0x60002), ("offsets", 0x20004),
                       ("ws", 0x50008)):
        rejected(bitmask_call(lib, **{name: P(addr)}), "aligned")


def test_bitmask_rejects_bad_outputs_and_workspace(lib):
    rejected(bitmask_call(lib, out_offsets=[0, 2]), "frame 1: output offset 2")
    rejected(bitmask_call(lib, out_offsets=[-4, 256]), "frame 0: output offset -4")
    rejected(bitmask_call(lib, out_bytes=256 + 63), "frame 1: output offset 256")
    rejected(bitmask_call(lib, out_offsets=[0, 252]), "the outputs of frames 0 and 1 overlap")
    rejected(bitmask_call(lib, out_offsets=[32, 0]), "the outputs of frames 0 and 1 overlap")
    need = lib.uc_bdd_bitmask_workspace_bytes
    need.restype = ctypes.c_long
    ints = lambda v: (ctypes.c_int * len(v))(*v)  # noqa: E731
    n = need(2, ints([2, 1]), ints([8, 4]), ints([8, 4]), ctypes.c_long(10))
    assert n > 4 * (8 * 8 + 4 * 4)
    rejected(bitmask_call(lib, ws_bytes=n - 1), "workspace too small")
    assert need(0, ints([1]), ints([1]), ints([1]), ctypes.c_long(0)) == -1
    assert need(1, ints([-1]), ints([1]), ints([1]), ctypes.c_long(0)) == -1
    assert need(1, ints([1]), ints([1]), ints([1]), ctypes.c_long(-1)) == -1
    # a frame without instances needs no winner map
    assert need(1, ints([0]), ints([720]), ints([1280]), ctypes.c_long(0)) < need(1, ints([1]), ints([720]), ints([1280]), ctypes.c_long(0)) - 4 * 720 * 1280 + 1

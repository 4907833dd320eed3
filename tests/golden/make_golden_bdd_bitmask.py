"""Golden fixture for the BDD100K MOTS bitmasks (qdtrack's seg_track format): runs the UNMODIFIED
external/qdtrack/qdtrack/core/to_bdd100k/utils.py (mask_prepare + mask_merge) on the CPU and reads every PNG it writes back.

    python tests/golden/make_golden_bdd_bitmask.py      (writes tests/golden/bdd_bitmask.npz; build container only)

pycocotools is absent, so pycocotools.mask.decode is stubbed to pass binary masks through (as make_golden_bdd.py does for encode):
the dicts given to mask_prepare hold the masks themselves, and the fixture stores their COCO strings (unicorn_b200.results.rle_encode,
checked to decode back to the mask) for the dicts the tests build.  SHAPE (hard-coded [720, 1280]) is set to each case's size.

Cases:
  tiny_*  the 8 MOTS frames of bdd_tiny_320.npz (288 x 320): the reference loop's track_result dicts (mots_tr_id / _bbox / _label /
          _row, the masks of mots_masks); bitmasks stored whole (tiny_bitmask).
  syn_*   synthetic frames at 720 x 1280 and at 1 x 1 and 7 x 13 (one without tracks), instances rasterised from stored parameters
          (syn_kind / syn_param: rectangle, ellipse, empty, full frame, seeded random bits): overlaps under distinct scores, ids 0, 255,
          256, 65535, 65536, labels 0..7 and a fractional label, masks whose first pixel is foreground, runs that cross column
          boundaries.  Equal scores only among instances that do not overlap, so numpy's order of ties does not show.  Bitmasks of
          up to SMALL pixels stored whole (syn_bitmask_<c>), the others as the sha256 of their bytes (syn_digest)."""
import hashlib
import importlib.util
import os
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from unicorn_b200.results import rle_decode, rle_encode  # noqa: E402

UTILS = os.path.join("/root/reference", "external", "qdtrack", "qdtrack", "core", "to_bdd100k", "utils.py")
SMALL = 1 << 12
RECT, ELLIPSE, EMPTY, FULL, RANDOM = 0, 1, 2, 3, 4


def rasterise(kind, p, h, w):
    """bool [h, w]: RECT p = (y0, x0, y1, x1) half-open; ELLIPSE centre (p0, p1), radii (p2, p3); RANDOM p0 = seed, p1 = percent on."""
    yy, xx = np.mgrid[:h, :w]
    if kind == RECT:
        return (yy >= p[0]) & (yy < p[2]) & (xx >= p[1]) & (xx < p[3])
    if kind == ELLIPSE:
        return ((yy - p[0]) / p[2]) ** 2 + ((xx - p[1]) / p[3]) ** 2 <= 1.0
    if kind == EMPTY:
        return np.zeros((h, w), dtype=bool)
    if kind == FULL:
        return np.ones((h, w), dtype=bool)
    return np.random.default_rng(int(p[0])).random((h, w)) < p[1] / 100.0


def synthetic_cases():
    """[(h, w, [(id, label, score, kind, params), ...]), ...]"""
    big = [  # 720 x 1280
        (65536, 0.0, 0.05, FULL, (0, 0, 0, 0)),  # the lowest score: the others paint over it
        (0, 1.0, 0.90, RECT, (0, 0, 200, 300)),  # first pixel foreground (a leading zero run)
        (255, 2.0, 0.40, ELLIPSE, (150, 250, 120, 180)),  # under id 0, over the full frame
        (256, 3.0, 0.95, ELLIPSE, (400, 600, 200, 250)),
        (65535, 4.0, 0.30, RECT, (0, 700, 720, 760)),  # full-height columns: runs across column boundaries
        (1, 5.0, 0.60, RECT, (650, 900, 720, 1100)),  # bottom rows, under nothing but the full frame
        (70000, 6.0, 0.60, RECT, (10, 1150, 100, 1270)),  # the same score as id 1, apart from it
        (12345, 7.0, 0.70, EMPTY, (0, 0, 0, 0)),
        (300, 0.0, 0.20, ELLIPSE, (719, 1279, 60, 90)),  # ends at the last pixel
        (9, 3.0, 0.99, RANDOM, (7, 5, 0, 0)),  # scattered pixels over everything
    ]
    rng = np.random.default_rng(11)
    crowd = []
    scores = rng.permutation(4000)[:40] / 4000.0 + 1e-3
    for n in range(40):
        cy, cx, ry, rx = rng.integers(0, 720), rng.integers(0, 1280), rng.integers(5, 150), rng.integers(5, 200)
        crowd.append((int(rng.integers(0, 1 << 20)), float(n % 8), float(scores[n]), ELLIPSE, (cy, cx, ry, rx)))
    one = [(5, 2.0, 0.5, FULL, (0, 0, 0, 0)), (6, 3.0, 0.7, FULL, (0, 0, 0, 0)), (7, 4.0, 0.6, EMPTY, (0, 0, 0, 0))]
    odd = [
        (256, 2.5, 0.3, RANDOM, (3, 50, 0, 0)),  # label + 1 = 3.5 is truncated
        (65535, 1.0, 0.8, RECT, (0, 0, 7, 1)),  # first column
        (65536, 0.0, 0.6, RANDOM, (4, 30, 0, 0)),
        (255, 7.0, 0.1, FULL, (0, 0, 0, 0)),
        (0, 6.0, 0.9, RECT, (5, 3, 7, 9)),  # rows 5-6 of columns 3-8: runs of two across columns
    ]
    return [(720, 1280, big), (720, 1280, crowd), (1, 1, one), (7, 13, odd), (7, 13, [])]


def tiny_frames(g):
    """Per MOTS frame of bdd_tiny_320.npz: [(id, bbox f32 [5], label f32, mask bool [h, w]), ...] in the dict's order."""
    h, w = (int(v) for v in g["orig"])
    masks = np.unpackbits(g["mots_masks"], axis=1, count=h * w).reshape(-1, h, w).astype(bool)
    starts = np.concatenate([[0], np.cumsum(g["mots_rows_n"])])
    t0 = np.concatenate([[0], np.cumsum(g["mots_tr_n"])])
    return [[(g["mots_tr_id"][j], g["mots_tr_bbox"][j], g["mots_tr_label"][j], masks[starts[f] + g["mots_tr_row"][j]])
             for j in range(t0[f], t0[f + 1])] for f in range(len(g["mots_tr_n"]))]


def load_utils():
    pkg = types.ModuleType("pycocotools")
    pkg.__path__ = []
    mask = types.ModuleType("pycocotools.mask")
    mask.decode = lambda m: np.asarray(m, dtype=np.uint8)  # the dicts hold the binary masks
    pkg.mask = mask
    sys.modules["pycocotools"], sys.modules["pycocotools.mask"] = pkg, mask
    spec = importlib.util.spec_from_file_location("qdtrack_to_bdd100k_utils", UTILS)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def reference_bitmask(utils, instances, h, w, tmp, name):
    """The PNG mask_merge writes for one frame, read back: uint8 [h, w, 4]."""
    from PIL import Image
    utils.SHAPE = [h, w]
    d = {np.int64(tid): dict(bbox=np.asarray(bbox, dtype=np.float32), label=np.float32(label), segm=m) for tid, bbox, label, m in instances}
    utils.mask_merge(utils.mask_prepare(d), name + ".jpg", tmp)
    im = Image.open(os.path.join(tmp, name + ".png"))
    assert im.mode == "RGBA" and im.size == (w, h)
    return np.asarray(im).copy()


def main():
    utils = load_utils()
    g = np.load(os.path.join(ROOT, "tests", "golden", "bdd_tiny_320.npz"))
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        h, w = (int(v) for v in g["orig"])
        tiny = [reference_bitmask(utils, fr, h, w, tmp, f"tiny{f}") for f, fr in enumerate(tiny_frames(g))]
        out["tiny_bitmask"] = np.stack(tiny)
        print("tiny: instances per frame", [len(fr) for fr in tiny_frames(g)], "painted pixels", [int((b != 0).any(-1).sum()) for b in tiny])
        hw, ks, ids, labels, scores, kinds, params, rles, digests = [], [], [], [], [], [], [], [], []
        for c, (h, w, insts) in enumerate(synthetic_cases()):
            frame = []
            for tid, label, score, kind, p in insts:
                m = rasterise(kind, p, h, w)
                s = rle_encode(m)
                assert np.array_equal(rle_decode(s, h, w), m)
                frame.append((tid, [0, 0, 0, 0, score], label, m))
                ids.append(tid)
                labels.append(label)
                scores.append(score)
                kinds.append(kind)
                params.append(p)
                rles.append(s)
            bm = reference_bitmask(utils, frame, h, w, tmp, f"syn{c}")
            hw.append((h, w))
            ks.append(len(insts))
            digests.append(hashlib.sha256(bm.tobytes()).hexdigest())
            if h * w <= SMALL:
                out[f"syn_bitmask_{c}"] = bm
            print(f"syn {c}: {h}x{w}, {len(insts)} instances, painted pixels {int((bm != 0).any(-1).sum())}, colours "
                  f"{len(np.unique(bm.reshape(-1, 4), axis=0))}")
    out.update(syn_hw=np.array(hw), syn_k=np.array(ks), syn_id=np.array(ids, dtype=np.int64), syn_label=np.array(labels, dtype=np.float32),
               syn_score=np.array(scores, dtype=np.float32), syn_kind=np.array(kinds), syn_param=np.array(params, dtype=np.int64),
               syn_rle=np.array(rles), syn_digest=np.array(digests))
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "bdd_bitmask.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()

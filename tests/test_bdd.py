"""The BDD100K test protocol without a GPU: the tracker settings, and the result builders (results.bbox2result / track2result /
segtrack2result / rle_dict) against the dicts of the unmodified qdtrack loop (tests/golden/bdd_tiny_320.npz, written by
tests/golden/make_golden_bdd.py): keys, per-class splits, shapes and dtypes, empty frames, and RLE dicts that decode to the golden's
masks."""
import json
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def load_bdd_golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "bdd_tiny_320.npz"))


def split(a, counts):
    """Rows of a stacked array back into consecutive groups of the given sizes."""
    off = np.concatenate([[0], np.cumsum(counts)])
    return [a[off[i]:off[i + 1]] for i in range(len(counts))]


def frames(g, p):
    """Per frame of branch p: (rows [n,7], ids, labels in the tracker's score order)."""
    return list(zip(split(g[p + "rows"], g[p + "rows_n"]), split(g[p + "ids"], g[p + "ids_n"]), split(g[p + "labels"], g[p + "ids_n"])))


def golden_bbox_result(g, p, f):
    per = split(g[p + "bbox"], g[p + "bbox_cls"].sum(1))[f]
    return split(per, g[p + "bbox_cls"][f])


def golden_masks(g):
    """Every MOTS detection's mask, bool [n, h, w], in NMS order."""
    h, w = (int(v) for v in g["orig"])
    return np.unpackbits(g["mots_masks"], axis=1, count=h * w).reshape(-1, h, w).astype(bool)


@pytest.fixture(scope="module")
def golden():
    return load_bdd_golden()


def tracked(g, p):
    """Per frame of branch p: the boxes the tracker returned (score order, duplicates removed), [k, 5]."""
    return split(g[p + "tboxes"], g[p + "ids_n"])


def test_bdd_tracker_has_the_qdtrack_config_values(golden):
    from unicorn_b200.tracker import bdd_tracker
    want = json.loads(str(golden["tracker_bdd"]))
    for mots, key in ((False, "mot"), (True, "mots")):
        t = bdd_tracker(mots, device="cpu")
        for k, v in want[key].items():
            assert getattr(t, k, "bisoftmax" if k == "match_metric" else None) == v, (key, k)
    lowered = json.loads(str(golden["lowered"]))
    for key in ("mot", "mots"):  # the golden ran the configs with only the lowered thresholds changed
        assert json.loads(str(golden[key + "_tracker_cfg"])) == dict(want[key], **lowered)


def test_bbox2result_per_class_in_nms_order(golden):
    from unicorn_b200.results import bbox2result
    for p in ("mot_", "mots_"):
        for f, (rows, _, _) in enumerate(frames(golden, p)):
            det = np.concatenate([rows[:, :4], rows[:, 4:5] * rows[:, 5:6]], 1)
            got = bbox2result(torch.from_numpy(det), torch.from_numpy(rows[:, 6]), int(golden["ncls"]))
            want = golden_bbox_result(golden, p, f)
            assert len(got) == len(want) == 8
            for a, b in zip(got, want):
                assert a.dtype == np.float32 and a.shape == b.shape and np.array_equal(a, b)


def test_track2result_rows_and_dtypes(golden):
    from unicorn_b200.results import track2result
    g = golden
    per_frame = split(g["mot_track"], g["mot_track_cls"].sum(1))
    for f, ((rows, ids, labels), boxes) in enumerate(zip(frames(g, "mot_"), tracked(g, "mot_"))):
        got = track2result(torch.from_numpy(boxes), torch.from_numpy(labels), torch.from_numpy(ids), 8)
        want = split(per_frame[f], g["mot_track_cls"][f])
        dtype = np.float64 if g["mot_track_f64"][f] else np.float32
        assert dtype == (np.float64 if (ids > -1).any() else np.float32)
        for a, b in zip(got, want):
            assert a.dtype == dtype and a.shape == b.shape and np.array_equal(a, b.astype(dtype))
    assert g["mot_track_f64"].any()


def test_empty_frames():
    from unicorn_b200.bdd import bdd_mot_result, bdd_mots_result
    r = bdd_mot_result(None, torch.zeros(0, 7), torch.zeros(0, 128), 1.0, 0, 8)
    assert set(r) == {"bbox_results", "track_results"}
    assert all(a.shape == (0, 5) and a.dtype == np.float32 for a in r["bbox_results"])
    assert all(a.shape == (0, 6) and a.dtype == np.float32 for a in r["track_results"])
    r = bdd_mots_result(None, torch.zeros(0, 7), torch.zeros(0, 128), 1.0, 0, [], 720, 1280, 8)
    assert set(r) == {"track_result", "bbox_result", "segm_result"} and len(r["track_result"]) == 0
    assert all(a.shape == (0, 5) and a.dtype == np.float32 for a in r["bbox_result"]) and r["segm_result"] == [[]] * 8


def test_track2result_without_valid_ids_is_float32():
    from unicorn_b200.results import track2result
    out = track2result(torch.rand(3, 5), torch.tensor([0.0, 1.0, 1.0]), torch.tensor([-1, -2, -1]), 8)
    assert len(out) == 8 and all(a.shape == (0, 6) and a.dtype == np.float32 for a in out)


def test_segtrack2result_and_rle_dicts_decode_to_the_golden_masks(golden):
    from unicorn_b200.results import rle_decode, rle_dict, rle_encode, segtrack2result
    g = golden
    h, w = (int(v) for v in g["orig"])
    masks = golden_masks(g)
    starts = np.concatenate([[0], np.cumsum(g["mots_rows_n"])])
    tr = split(np.arange(len(g["mots_tr_id"])), g["mots_tr_n"])
    valids = split(g["mots_valids"], g["mots_rows_n"])
    for f, ((rows, ids, labels), boxes) in enumerate(zip(frames(g, "mots_"), tracked(g, "mots_"))):
        fm = masks[starts[f]:starts[f + 1]]
        segms = [rle_dict(rle_encode(fm[r]), h, w) for r in np.flatnonzero(valids[f])]  # masks_full[indexs]
        got = segtrack2result(torch.from_numpy(boxes), torch.from_numpy(labels), segms, torch.from_numpy(ids))
        want = tr[f]
        assert [type(k) for k in got] == [np.int64] * len(want) and list(got) == g["mots_tr_id"][want].tolist()
        for j, (tid, v) in zip(want, got.items()):
            assert v["bbox"].dtype == np.float32 and np.array_equal(v["bbox"], g["mots_tr_bbox"][j])
            assert v["label"].dtype == np.float32 and v["label"] == g["mots_tr_label"][j]
            assert v["segm"]["size"] == [h, w] and isinstance(v["segm"]["counts"], bytes)
            assert np.array_equal(rle_decode(v["segm"]["counts"].decode(), h, w), fm[g["mots_tr_row"][j]])

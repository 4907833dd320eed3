"""The COCO instance segmenter (unicorn_inst_convnext_tiny) off the GPU: the weight table against the reference's manifest, checkpoints
of the detector and of the tracking mask models, the shim's Exp, the oracle's mask head and postprocess_inst against the reference
golden (tests/golden/inst_tiny_320.npz, with the decoded head of det_tiny_320.npz), the COCO result format, and the argument checks
of uc_inst_encode_batched."""
import ctypes
import json
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

from unicorn_b200.weights import CONFIGS, check_state_dict, make_state_dict, param_shapes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
INST = "unicorn_inst_convnext_tiny"


def load_inst_golden():
    """tests/golden/inst_tiny_320.npz as a dict, with its JSON text unpacked (rles, orig_rles, coco) and the decoded head, which is
    det_tiny_320.npz's (the same frame, and make_state_dict gives the shared parameters the detector's values)."""
    g = dict(np.load(os.path.join(GOLD, "inst_tiny_320.npz")))
    g.update(json.loads(bytes(g.pop("text")).decode()))
    g["head"] = np.load(os.path.join(GOLD, "det_tiny_320.npz"))["head"]
    g["fpn_levels"] = g["fpn_levels"].astype(np.int64)
    return g


def test_inst_param_shapes_match_reference_manifest():
    man = json.load(open(os.path.join(GOLD, f"manifest_{INST}.json")))
    assert [(k, list(v)) for k, v in param_shapes(INST).items()] == list(man.items())
    cfg = CONFIGS[INST]
    assert cfg["task"] == "det" and cfg["num_classes"] == 80 and cfg["mask"] and cfg["dims"] == CONFIGS["unicorn_det_convnext_tiny"]["dims"]
    S, D = param_shapes(INST), param_shapes("unicorn_det_convnext_tiny")
    extra = [k for k in S if k not in D]
    assert all(S[k] == v for k, v in D.items())  # the detector's key set, plus the mask keys
    assert extra and all(k.startswith(("head.controllers.", "head.mask_branch.", "head.mask_head.")) for k in extra)
    assert S["head.controllers.0.weight"] == (169, 256, 3, 3)


@pytest.mark.parametrize("other", ["unicorn_det_convnext_tiny", "unicorn_track_tiny_mask"])
def test_inst_state_dict_and_cross_rejection(other):
    check_state_dict(make_state_dict(INST, 0), INST)
    with pytest.raises(ValueError, match="does not match"):
        check_state_dict(make_state_dict(other, 0), INST)
    with pytest.raises(ValueError, match="does not match"):
        check_state_dict(make_state_dict(INST, 0), other)


def test_shim_serves_the_inst_exp():
    code = textwrap.dedent(f"""
        import sys
        sys.path.insert(0, {ROOT!r})
        import unicorn_b200.shim as shim
        shim.install()
        import torch
        from unicorn.exp import get_exp, ExpDet, ExpDetMask
        from unicorn_b200.weights import make_state_dict
        exp = get_exp("exps/default/unicorn_inst_convnext_tiny_800x1280.py", None)
        assert isinstance(exp, ExpDetMask) and isinstance(exp, ExpDet)
        assert exp.task == "inst" and exp.num_classes == 80 and exp.d_rate == 2 and exp.use_raft and exp.ctrl_loc == "reg"
        assert exp.test_conf == 0.01 and exp.nmsthre == 0.65 and exp.mask_thres == 0.3 and exp.test_size == (800, 1280)
        assert exp.backbone_name == "convnext" and exp.in_channels == [192, 384, 768] and exp.mask
        model = exp.get_model(load_pretrain=False)
        assert model.head.mask_head is not None and model.num_classes == 80
        r = model.load_state_dict(make_state_dict("unicorn_inst_convnext_tiny", 0), strict=True)
        assert not r.missing_keys and not r.unexpected_keys
        for other in ("unicorn_det_convnext_tiny", "unicorn_track_tiny_mask"):
            try:
                model.load_state_dict(make_state_dict(other, 0)); raise SystemExit(other + " checkpoint accepted")
            except RuntimeError:
                pass
        assert get_exp("exps/default/unicorn_det_convnext_tiny_800x1280.py", None).mask_thres == 0.3
        print("inst shim ok")
    """)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "inst shim ok" in r.stdout, r.stdout + r.stderr


def test_oracle_inst_head_and_postprocess_match_reference_golden():
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import unicorn_oracle as orc
    from unicorn_b200.results import rle_decode
    from unicorn_b200.synthetic import make_video
    g = load_inst_golden()
    frames, _ = make_video(2, 320, 320, seed=int(g["seed_video"]), n_obj=int(g["n_obj"]))
    f = int(g["frame"])
    sd = make_state_dict(INST, 0)
    sd.update({f"head.beta_{k}": torch.zeros(256, 1, 1) for k in range(3)})  # zero prior: x + 0 * beta == x
    sd.update({f"pos_emb.{a}_embed.weight": torch.zeros(40, 128) for a in ("row", "col")})  # only feeds the unused sequence dict
    with torch.no_grad():
        out6 = orc.whole_forward(frames[f:f + 1], sd, dict(CONFIGS[INST]))[0]
    out, locs, dyn, lvls, mf, um = out6
    rel = lambda a, b: ((a - b).abs().max() / (b.abs().max() + 1e-12)).item()  # noqa: E731
    assert out.shape == (1, 2100, 85) and rel(out, torch.from_numpy(g["head"])) < 1e-4
    assert torch.equal(locs, torch.from_numpy(g["locations"])) and torch.equal(lvls, torch.from_numpy(g["fpn_levels"]))
    assert rel(dyn[0, ::16], torch.from_numpy(g["dyn_sub"])) < 1e-4
    assert rel(mf, torch.from_numpy(g["mask_feats"])) < 1e-4 and rel(um[0, :, ::4, ::4], torch.from_numpy(g["up_masks_sub"])) < 1e-4
    dets, masks = orc.postprocess_inst(*out6, 80, float(g["conf"]), float(g["nms"]), d_rate=int(g["d_rate"]))
    want = torch.from_numpy(g["dets"])
    assert dets.shape == want.shape and 20 <= dets.shape[0] <= 200 and torch.equal(dets[:, 6], want[:, 6])
    assert (dets - want).abs().max() < 1e-4
    assert (masks[:8, 0, ::4, ::4] - torch.from_numpy(g["soft_sub"]).float()).abs().max() < 1e-3  # fp16 storage
    thr = float(g["thr"])
    # a pixel within 1e-5 of the threshold may flip between two fp32 evaluations of the same mask; no other may
    for s, m in zip(g["rles"], masks[:, 0]):
        diff = torch.from_numpy(rle_decode(s, 320, 320)) != (m > thr)
        assert not diff[(m - thr).abs() >= 1e-5].any()


def _golden_coco():
    g = load_inst_golden()
    h, w = (int(v) for v in g["orig"])
    return g, h, w, min(320 / float(h), 320 / float(w)), [int(c) for c in g["class_ids"]]


def test_coco_instances_polygons_match_reference_format():
    from unicorn_b200.results import coco_instances
    g, h, w, r, class_ids = _golden_coco()
    assert g["coco"]  # the golden's original size shortens the resize: the masks' last row is padding
    got = coco_instances(torch.from_numpy(g["dets"]), list(g["orig_rles"]), r, h, w, int(g["image_id"]), class_ids)
    assert got == g["coco"]


def test_coco_instances_rle_mode_decodes_to_the_masks():
    from unicorn_b200.results import coco_detections, coco_instances, rle_decode, rle_encode
    g, h, w, r, class_ids = _golden_coco()
    rles = list(g["orig_rles"])
    rles[3] = rle_encode(np.zeros((h, w), dtype=bool))  # an empty mask is dropped
    got = coco_instances(torch.from_numpy(g["dets"]), rles, r, h, w, 7, class_ids, polygons=False)
    base = coco_detections(torch.from_numpy(g["dets"]), r, 7, class_ids)
    keep = [i for i in range(len(rles)) if i != 3]
    assert len(got) == len(keep)
    for d, i in zip(got, keep):
        assert d["segmentation"]["size"] == [h, w] and d["segmentation"]["counts"] == rles[i]
        assert {k: v for k, v in d.items() if k != "segmentation"} == {k: v for k, v in base[i].items() if k != "segmentation"}
        assert np.array_equal(rle_decode(d["segmentation"]["counts"], h, w), rle_decode(g["orig_rles"][i], h, w))


# ---- uc_inst_encode_batched: every call below is rejected before anything is launched (fake, never dereferenced pointers)
P = ctypes.c_void_p
EINVAL = -1
A16 = [P(0x10000 * (i + 1)) for i in range(8)]


@pytest.fixture(scope="module")
def lib():
    from unicorn_b200 import _lib
    L = _lib.lib()
    L.uc_mots_encode_workspace_bytes.restype = ctypes.c_long
    return L


def enc(lib, maps=A16[0], bs=None, n_max=4, hs=40, ws=64, d_rate=2, B=2, count=A16[1], row0=0, H=(100, 120), W=(160, 90),
        r=(0.8, 0.8), work=A16[2], work_bytes=None, emit=A16[3], chars=A16[4], capacity=1024, offsets=A16[5]):
    if bs is None:
        bs = n_max * hs * ws
    if work_bytes is None:
        work_bytes = lib.uc_mots_encode_workspace_bytes(max(B, 1) * n_max, max(H or (1,)), max(W or (1,)))
    rc = lib.uc_inst_encode_batched(maps, ctypes.c_long(bs), n_max, hs, ws, d_rate, B, count, row0,
                                    (ctypes.c_int * len(H))(*H) if H is not None else None, (ctypes.c_int * len(W))(*W),
                                    (ctypes.c_double * len(r))(*r), ctypes.c_float(0.3), work, ctypes.c_long(work_bytes), emit, chars,
                                    ctypes.c_long(capacity), offsets, None)
    return rc, lib.uc_last_error()


def rejected(call, *words):
    rc, msg = call
    assert rc == EINVAL, (rc, msg)
    for w in words:
        assert w.encode() in msg, (w, msg)


def test_inst_encode_symbol_is_exported(lib):
    assert hasattr(lib, "uc_inst_encode_batched")


def test_inst_encode_rejects_bad_arguments(lib):
    rejected(enc(lib, H=None), "uc_inst_encode_batched", "null pointer")
    rejected(enc(lib, B=0, H=(), W=(), r=()), "B = 0 must be in 1..64")
    rejected(enc(lib, B=65, H=(100,) * 65, W=(100,) * 65, r=(1.0,) * 65), "B = 65 must be in 1..64")
    for k in ("maps", "count", "work", "emit", "offsets"):
        rejected(enc(lib, **{k: None}), "null pointer")
    rejected(enc(lib, chars=None), "null pointer")
    rejected(enc(lib, n_max=0), "bad sizes")
    rejected(enc(lib, hs=0), "bad sizes")
    rejected(enc(lib, d_rate=0), "bad sizes")
    rejected(enc(lib, n_max=40000, bs=40000 * 40 * 64), "slots must be <= 65535")
    rejected(enc(lib, row0=-1), "row0 = -1 must be >= 0")
    rejected(enc(lib, bs=4 * 40 * 64 - 1), "bad per-image stride")
    rejected(enc(lib, H=(100, 0)), "image 1: bad sizes")
    rejected(enc(lib, r=(0.8, 0.0)), "image 1: bad sizes")
    rejected(enc(lib, capacity=-1), "negative capacity")
    rejected(enc(lib, maps=P(0x10002)), "aligned")
    rejected(enc(lib, offsets=P(0x10004)), "aligned")
    rejected(enc(lib, work=P(0x10008)), "aligned")
    rejected(enc(lib, r=(0.8, 1e6)), "image 1: the resized mask is empty")
    rejected(enc(lib, work_bytes=1024), "workspace too small")
    rejected(enc(lib, H=(100, 1 << 22), W=(160, 1 << 20)), "image 1: frame too large")

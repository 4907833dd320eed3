"""The COCO detectors (unicorn_det_convnext_tiny / _large / _r50) off the GPU: the weight table against the reference's manifests,
cross-task checkpoints, the oracle's prior-less head against the reference goldens, the shim's Exp / model surface, the COCO result
format, and the argument checks of the detector's C entry points."""
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
DET = ("unicorn_det_convnext_tiny", "unicorn_det_convnext_large", "unicorn_det_r50")


@pytest.mark.parametrize("name", DET)
def test_det_param_shapes_match_reference_manifest(name):
    man = json.load(open(os.path.join(GOLD, f"manifest_{name}.json")))
    assert [(k, list(v)) for k, v in param_shapes(name).items()] == list(man.items())
    cfg = CONFIGS[name]
    assert cfg["task"] == "det" and cfg["num_classes"] == 80 and not cfg["mask"]
    S = param_shapes(name)
    assert S["head.cls_preds.0.weight"] == (80, 256, 1, 1)
    assert not any(k.startswith(("head.beta_", "bottleneck", "upsample_layer", "transformer", "pos_emb")) or "_sot." in k for k in S)


@pytest.mark.parametrize("det,track", [("unicorn_det_convnext_tiny", "unicorn_track_tiny"), ("unicorn_det_convnext_large", "unicorn_track_large"),
                                       ("unicorn_det_r50", "unicorn_track_r50")])
def test_det_state_dict_and_cross_task_rejection(det, track):
    check_state_dict(make_state_dict(det, 0), det)
    with pytest.raises(ValueError, match="does not match"):
        check_state_dict(make_state_dict(track, 0), det)
    with pytest.raises(ValueError, match="does not match"):
        check_state_dict(make_state_dict(det, 0), track)
    # the backbone and neck of a detector are those of the tracking model of the same backbone
    st, sd = param_shapes(track), param_shapes(det)
    assert all(st[k] == v for k, v in sd.items() if k.startswith("backbone."))


def _oracle_head(img, name):
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import resnet_oracle as ro
    import unicorn_oracle as orc
    sd = make_state_dict(name, 0)
    sd.update({f"head.beta_{k}": torch.zeros(256, 1, 1) for k in range(3)})  # zero prior: x + 0 * beta == x
    sd.update({f"pos_emb.{a}_embed.weight": torch.zeros(40, 128) for a in ("row", "col")})  # only feeds the unused sequence dict
    fwd = ro.whole_forward if CONFIGS[name]["backbone"] == "resnet50" else orc.whole_forward
    return fwd(img, sd, dict(CONFIGS[name]))[0], orc


@pytest.mark.parametrize("tag,name", [("tiny", "unicorn_det_convnext_tiny"), ("r50", "unicorn_det_r50"), ("large", "unicorn_det_convnext_large")])
def test_oracle_det_forward_matches_reference_golden(tag, name):
    from unicorn_b200.synthetic import make_video
    g = np.load(os.path.join(GOLD, f"det_{tag}_320.npz"))
    frames, _ = make_video(2, 320, 320, seed=int(g["seed_video"]), n_obj=int(g["n_obj"]))
    f = int(g["frame"])
    with torch.no_grad():
        head, orc = _oracle_head(frames[f:f + 1], name)
    ref = torch.from_numpy(g["head"])
    assert head.shape == ref.shape == (1, 2100, 85)
    assert ((head - ref).abs().max() / ref.abs().max()).item() < 1e-4
    dets = orc.postprocess(ref.clone(), 80, float(g["conf"]), float(g["nms"]))[0]
    want = torch.from_numpy(g["dets"])
    assert dets.shape == want.shape and torch.equal(dets[:, 6], want[:, 6])
    assert (dets[:, :6] - want[:, :6]).abs().max() < 1e-4


def test_oracle_agnostic_nms_matches_reference_golden():
    """Class-agnostic rows of the reference (torchvision.ops.nms) are the oracle's greedy NMS over all candidates."""
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import unicorn_oracle as orc
    g = np.load(os.path.join(GOLD, "det_tiny_320.npz"))
    dets = agnostic_reference(orc, torch.from_numpy(g["head"])[0], float(g["conf_agnostic"]), float(g["nms_agnostic"]))
    want = torch.from_numpy(g["dets_agnostic"])
    assert dets.shape == want.shape and torch.equal(dets[:, 6], want[:, 6]) and (dets[:, :6] - want[:, :6]).abs().max() < 1e-4


def agnostic_reference(orc, pred, conf, nms):
    """postprocess(..., class_agnostic=True) of one image's decoded rows [A, 5+ncls] with the oracle's greedy NMS."""
    p = pred.clone()
    box = torch.stack([p[:, 0] - p[:, 2] / 2, p[:, 1] - p[:, 3] / 2, p[:, 0] + p[:, 2] / 2, p[:, 1] + p[:, 3] / 2], 1)
    cc, cp = torch.max(p[:, 5:], 1, keepdim=True)
    det = torch.cat([box, p[:, 4:5], cc, cp.float()], 1)[p[:, 4] * cc[:, 0] >= conf]
    keep = orc.nms_greedy(det[:, :4].numpy(), (det[:, 4] * det[:, 5]).numpy(), nms)
    return det[torch.from_numpy(keep)]


def test_coco_detections_match_reference_format():
    from unicorn_b200.results import coco_detections
    g = json.load(open(os.path.join(GOLD, "coco_detections.json")))
    H, W = g["img_size"]
    got = []
    for (h, w, img_id), rows in zip(g["images"], g["rows"]):
        r = min(H / float(h), W / float(w))
        got += coco_detections(torch.tensor(rows, dtype=torch.float32), r, img_id, g["class_ids"])
    assert got == g["coco"]
    assert coco_detections(None, 1.0, 0, g["class_ids"]) == []


def test_shim_serves_the_det_exps():
    code = textwrap.dedent(f"""
        import sys
        sys.path.insert(0, {ROOT!r})
        import unicorn_b200.shim as shim
        shim.install()
        import inspect
        import torch
        from unicorn.exp import get_exp
        from unicorn.utils import postprocess
        from unicorn_b200.weights import make_state_dict
        from unicorn_b200._lib import UnicornB200Error
        assert "class_agnostic" in inspect.signature(postprocess).parameters
        for f, name, bb, inc in (("unicorn_det_convnext_tiny_800x1280", "unicorn_det_convnext_tiny", "convnext", [192, 384, 768]),
                                 ("unicorn_det_convnext_large_800x1280", "unicorn_det_convnext_large", "convnext_large", [384, 768, 1536]),
                                 ("unicorn_det_r50_800x1280", "unicorn_det_r50", "resnet50", [512, 1024, 2048])):
            exp = get_exp(f"exps/default/{{f}}.py", None)
            assert exp.num_classes == 80 and exp.test_size == (800, 1280) and exp.test_conf == 0.01 and exp.nmsthre == 0.65
            assert exp.backbone_name == bb and exp.in_channels == inc, (exp.backbone_name, exp.in_channels)
            model = exp.get_model(load_pretrain=False)
            assert model.head.decode_in_inference and model.eval() is model and model.half() is model
            r = model.load_state_dict(make_state_dict(name, 0), strict=True)
            assert not r.missing_keys and not r.unexpected_keys
            try:
                model.load_state_dict(make_state_dict("unicorn_track_tiny", 0)); raise SystemExit("tracking checkpoint accepted")
            except RuntimeError:
                pass
            try:
                model(torch.zeros(1, 3, 32, 32)); raise SystemExit("ran without a GPU engine")
            except RuntimeError:
                pass
            if not torch.cuda.is_available():
                try:
                    model.cuda(); raise SystemExit("built an engine without a GPU")
                except UnicornB200Error:
                    pass
        print("det shim ok")
    """)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "det shim ok" in r.stdout, r.stdout + r.stderr


# ---- C entry points: every call below is rejected before anything is launched (fake, never dereferenced pointers)
P = ctypes.c_void_p
EINVAL = -1
A16 = [P(0x10000 * (i + 1)) for i in range(8)]


@pytest.fixture(scope="module")
def lib():
    from unicorn_b200 import _lib
    L = _lib.lib()
    L.uc_postprocess_workspace_bytes_batched.restype = ctypes.c_long
    return L


def test_det_symbols_are_exported(lib):
    for s in ("uc_det_candidates_batched", "uc_postprocess_nms_batched", "uc_postprocess_batched_ex"):
        assert hasattr(lib, s), s


def _levels(hw=(40, 40, 20, 20, 10, 10)):
    return ((P * 3)(*A16[:3]), (P * 3)(*A16[3:6]), (ctypes.c_int * 6)(*hw), (ctypes.c_int * 3)(8, 16, 32))


def cand(lib, ld_ro=8, ld_cls=80, ncls=80, B=2, ws=A16[6], ws_bytes=None, bs=True, hw=(40, 40, 20, 20, 10, 10)):
    ro, cl, hwa, st = _levels(hw)
    A = hw[0] * hw[1] + hw[2] * hw[3] + hw[4] * hw[5]
    if ws_bytes is None:
        ws_bytes = lib.uc_postprocess_workspace_bytes_batched(A, max(B, 1))
    bro = (ctypes.c_long * 3)(*[hw[2 * k] * hw[2 * k + 1] * ld_ro for k in range(3)]) if bs else None
    bcl = (ctypes.c_long * 3)(*[hw[2 * k] * hw[2 * k + 1] * ld_cls for k in range(3)]) if bs else None
    rc = lib.uc_det_candidates_batched(ro, cl, hwa, st, ld_ro, ld_cls, bro, bcl, ncls, B, ctypes.c_float(0.01), ws, ctypes.c_long(ws_bytes), None)
    return rc, lib.uc_last_error()


def rejected(call, *words):
    rc, msg = call
    assert rc == EINVAL, (rc, msg)
    for w in words:
        assert w.encode() in msg, (w, msg)


def test_det_candidates_rejects_bad_arguments(lib):
    rejected(cand(lib, ncls=0), "uc_det_candidates_batched", "bad arguments")
    rejected(cand(lib, ncls=81), "bad arguments")            # more classes than columns
    rejected(cand(lib, ld_ro=4), "bad arguments")            # reg + obj need 5 columns
    rejected(cand(lib, B=0), "B must be >= 1")
    rejected(cand(lib, ws=None), "null workspace")
    rejected(cand(lib, bs=False), "null per-image strides")
    rejected(cand(lib, ws_bytes=1024), "workspace too small")


def nms(lib, A=2100, B=2, flags=0, ws=A16[6], ws_bytes=None, dets=A16[7], count=A16[0]):
    if ws_bytes is None:
        ws_bytes = lib.uc_postprocess_workspace_bytes_batched(A, max(B, 1))
    rc = lib.uc_postprocess_nms_batched(A, ctypes.c_float(0.65), 0, B, flags, ws, ctypes.c_long(ws_bytes), dets, count, None, None)
    return rc, lib.uc_last_error()


def test_postprocess_nms_rejects_bad_arguments(lib):
    rejected(nms(lib, flags=2), "uc_postprocess_nms_batched", "unknown flags")
    rejected(nms(lib, A=0), "bad arguments")
    rejected(nms(lib, ws=None), "bad arguments")
    rejected(nms(lib, dets=None), "bad arguments")
    rejected(nms(lib, B=0), "B must be >= 1")
    rejected(nms(lib, ws_bytes=64), "workspace too small")


def test_postprocess_ex_rejects_bad_arguments(lib):
    def ex(pred=A16[1], A=2100, ncls=80, B=1, flags=1, ws_bytes=None):
        if ws_bytes is None:
            ws_bytes = lib.uc_postprocess_workspace_bytes_batched(A, max(B, 1))
        rc = lib.uc_postprocess_batched_ex(pred, A, ncls, ctypes.c_float(0.01), ctypes.c_float(0.65), 0, B, flags, A16[6], ctypes.c_long(ws_bytes),
                                           A16[7], A16[0], None, None)
        return rc, lib.uc_last_error()
    rejected(ex(flags=4), "uc_postprocess_batched_ex", "unknown flags")
    rejected(ex(pred=None), "bad arguments")
    rejected(ex(ncls=0), "bad arguments")
    rejected(ex(B=0), "B must be >= 1")
    rejected(ex(ws_bytes=64), "workspace too small")

"""Golden fixture of the COCO instance segmenter (exps/default/unicorn_inst_convnext_tiny_800x1280.py: YOLOX + YOLOXHeadDetMask,
CondInst with the RAFT upsampler, d_rate 2) from the UNMODIFIED reference, and a check of the oracle against it.

    python tests/golden/make_golden_inst.py      (writes tests/golden/inst_tiny_320.npz; build container only)

Stored for the seeded synthetic 320x320 frame of det_tiny_320.npz with make_state_dict("unicorn_inst_convnext_tiny", 0):
  - the 6-tuple of `model(imgs)` except the decoded head: it is the head of det_tiny_320.npz (make_state_dict seeds every
    parameter by its name, so the shared backbone, neck and head get the detector's weights; asserted below).  locations,
    fpn_levels and mask_feats in full; the controller outputs at every 16th anchor (dyn_sub) and the up-masks at every 4th pixel
    in each direction (up_masks_sub);
  - the rows of `postprocess_inst` at the evaluator's NMS threshold 0.65 and conf CONF = 0.04 (59 rows).  With seeded weights the
    evaluator's conf 0.01 leaves 1528 of the 2100 anchors; 0.04 keeps the fixture small;
  - the soft masks of the first 8 rows at every 4th pixel in each direction (soft_sub, fp16);
  - per row, the fraction of the network-input mask's pixels within 0.05 of the threshold (near_thr): the seeded weights give some
    rows flat masks whose thresholded area a small change of the logits moves a lot;
  - as UTF-8 JSON (text): the masks of all rows thresholded at 0.3 as COCO RLE strings, at the network input (rles) and as the
    evaluator resizes them to ORIG, padded with background to the whole ORIG frame (orig_rles); and
    COCOInstEvaluator.convert_to_coco_format (mask_thres 0.3, as exp/unicorn_det.py:92 sets it) of those rows and masks for
    one original size ORIG whose floor rule makes the resized mask one row shorter than the image, with a stub dataset holding the
    COCO class_ids (coco)."""
import importlib.util
import json
import math
import os
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
HERE = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, HERE)
import ref_import  # noqa: E402
import unicorn_oracle as orc  # noqa: E402
from make_golden_coco import CLASS_IDS  # noqa: E402
from unicorn_b200.results import rle_encode  # noqa: E402
from unicorn_b200.synthetic import make_video  # noqa: E402
from unicorn_b200.weights import CONFIGS, make_state_dict  # noqa: E402

NAME, H, W = "unicorn_inst_convnext_tiny", 320, 320
CONF, NMS, THR, D_RATE, KEEP = 0.04, 0.65, 0.3, 2, 8


def shortened_size():
    """The first original (h, w) with h > w >= 200 whose resized mask is shorter than h (floor(320 * (1 / (320 / h))) < h)."""
    for h in range(321, 2000):
        for w in range(200, h):
            s = min(H / float(h), W / float(w))
            if math.floor(H * (1 / s)) < h and math.floor(W * (1 / s)) >= w:
                return h, w
    raise AssertionError("no shortened size")


def oracle_forward(img, sd):
    """The oracle's whole-mode mask head (zero priors) on the instance-segmenter weights."""
    sd = dict(sd, **{f"head.beta_{k}": torch.zeros(256, 1, 1) for k in range(3)},
              **{f"pos_emb.{a}_embed.weight": torch.zeros(40, 128) for a in ("row", "col")})
    return orc.whole_forward(img, sd, dict(CONFIGS[NAME]))[0]


def main():
    ref_import.install()
    frames, _ = make_video(2, H, W, seed=1, n_obj=3)
    img = frames[1:2]
    sd = make_state_dict(NAME, 0)
    exp, model = ref_import.get_model(NAME + "_800x1280")
    assert exp.task == "inst" and exp.d_rate == D_RATE and exp.use_raft and exp.mask_thres == THR
    print(model.load_state_dict(sd, strict=True))
    from unicorn.utils.boxes import postprocess_inst
    with torch.no_grad():
        out6 = tuple(t.clone() for t in model(img))
        outs, locs, dyn, lvls, mf, um = (t.clone() for t in out6)  # postprocess_inst turns outs into corners in place
        dets, masks = postprocess_inst(outs, locs, dyn, lvls, mf, model.head.mask_head, 80, CONF, NMS, d_rate=D_RATE, up_masks=um)
        dets, masks = dets[0], masks[0]
    print("rows", dets.shape[0], "masks", tuple(masks.shape))
    assert 20 <= dets.shape[0] <= 200
    o6 = oracle_forward(img, sd)
    for a, b, n in zip(o6, out6, ("outputs", "locations", "dyn", "levels", "mask_feats", "up_masks")):
        err = ((a.float() - b.float()).abs().max() / (b.float().abs().max() + 1e-12)).item()
        print(f"{n:10s} oracle-vs-reference rel err {err:.3e}")
        assert err < 1e-4
    od, om = orc.postprocess_inst(*out6, 80, CONF, NMS, d_rate=D_RATE)
    assert torch.equal(od[:, 6], dets[:, 6]) and (od - dets).abs().max() < 1e-4 and (om - masks).abs().max() < 1e-4

    spec = importlib.util.spec_from_file_location("coco_inst_evaluator", os.path.join(ref_import.REF_ROOT, "unicorn", "evaluators",
                                                                                      "coco_inst_evaluator.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    ev = object.__new__(mod.COCOInstEvaluator)
    ev.img_size, ev.mask_thres = (H, W), THR
    ev.dataloader = types.SimpleNamespace(dataset=types.SimpleNamespace(class_ids=CLASS_IDS))
    orig = shortened_size()
    coco = ev.convert_to_coco_format([dets.clone()], [masks.clone()], ([orig[0]], [orig[1]]), [42])
    print("original size", orig, "coco dicts", len(coco), "of", dets.shape[0])
    rles = [rle_encode(m.numpy()) for m in (masks[:, 0] > THR)]
    near_thr = ((masks[:, 0] - THR).abs() < 0.05).float().mean(dim=(1, 2))
    s = min(H / float(orig[0]), W / float(orig[1]))
    ori = F.interpolate(masks, scale_factor=1 / s, mode="bilinear", align_corners=False)[:, 0, :orig[0], :orig[1]] > THR
    assert ori.shape[1] < orig[0]
    full = torch.zeros(ori.shape[0], *orig, dtype=torch.bool)
    full[:, :ori.shape[1], :ori.shape[2]] = ori
    orig_rles = [rle_encode(m.numpy()) for m in full]
    det = np.load(os.path.join(HERE, "det_tiny_320.npz"))
    assert int(det["seed_video"]) == 1 and int(det["n_obj"]) == 3 and int(det["frame"]) == 1
    assert np.array_equal(det["head"], out6[0].numpy())
    text = json.dumps(dict(rles=rles, orig_rles=orig_rles, coco=coco))
    np.savez_compressed(os.path.join(HERE, "inst_tiny_320.npz"), locations=locs.numpy(), dyn_sub=dyn[0, ::16].numpy(),
                        fpn_levels=lvls.numpy().astype(np.int8), mask_feats=mf.numpy(), up_masks_sub=um[0, :, ::4, ::4].numpy(),
                        dets=dets.numpy(), soft_sub=masks[:KEEP, 0, ::4, ::4].numpy().astype(np.float16), near_thr=near_thr.numpy(),
                        text=np.frombuffer(text.encode(), dtype=np.uint8), conf=CONF, nms=NMS, thr=THR, d_rate=D_RATE, seed_video=1,
                        n_obj=3, frame=1, orig=np.array(orig), image_id=42, class_ids=np.array(CLASS_IDS))

if __name__ == "__main__":
    main()

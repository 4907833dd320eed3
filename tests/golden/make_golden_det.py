"""Golden fixtures of the COCO detectors (exps/default/unicorn_det_*_800x1280.py: YOLOX + YOLOXHeadDet) from the UNMODIFIED
reference, and a check of the oracle's prior-less head against them.

    python tests/golden/make_golden_det.py      (writes tests/golden/det_{tiny,r50,large}_320.npz; build container only)

Stored per model: the decoded head output of `model(imgs)` for a seeded synthetic 320x320 frame (80 classes -> 85 columns) and the
rows of `postprocess` class-aware at the evaluator's thresholds (conf 0.01, nms 0.65) and class-agnostic at the NMS threshold of
tools/demo.py (0.3).  The agnostic rows use conf 0.01 rather than the demo's 0.3: no score of the seeded weights reaches 0.3.  The oracle runs the head of the tracking models with zero priors: a detector state_dict plus zero
`beta_*` scales is the same network."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
HERE = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, HERE)
import ref_import  # noqa: E402
import resnet_oracle as ro  # noqa: E402
import unicorn_oracle as orc  # noqa: E402
from make_golden_r50 import install_offline_resnet  # noqa: E402
from unicorn_b200.synthetic import make_video  # noqa: E402
from unicorn_b200.weights import CONFIGS, make_state_dict  # noqa: E402

H = W = 320
AWARE, AGNOSTIC = (0.01, 0.65), (0.01, 0.3)
MODELS = (("tiny", "unicorn_det_convnext_tiny"), ("r50", "unicorn_det_r50"), ("large", "unicorn_det_convnext_large"))


def oracle_head(img, sd, name):
    """The oracle's whole-mode forward (zero priors) on the detector weights: the prior term is x + 0 * beta; the position table
    only feeds the unused sequence dict."""
    sd = dict(sd, **{f"head.beta_{k}": torch.zeros(256, 1, 1) for k in range(3)},
              **{f"pos_emb.{a}_embed.weight": torch.zeros(40, 128) for a in ("row", "col")})
    cfg = dict(CONFIGS[name])
    fwd = ro.whole_forward if cfg["backbone"] == "resnet50" else orc.whole_forward
    return fwd(img, sd, cfg)[0]


def main():
    install_offline_resnet()
    frames, _ = make_video(2, H, W, seed=1, n_obj=3)
    img = frames[1:2]
    from unicorn.utils.boxes import postprocess
    for tag, name in MODELS:
        sd = make_state_dict(name, 0)
        _, model = ref_import.get_model(name + "_800x1280")
        print(model.load_state_dict(sd, strict=True))
        with torch.no_grad():
            head = model(img)
            aware = postprocess(head.clone(), 80, *AWARE)[0]
            agnostic = postprocess(head.clone(), 80, *AGNOSTIC, class_agnostic=True)[0]
        o_head = oracle_head(img, sd, name)
        e = ((o_head - head).abs().max() / head.abs().max()).item()
        print(name, "head oracle-vs-reference rel err", e, "rows", aware.shape[0], agnostic.shape[0])
        assert e < 1e-4
        np.savez_compressed(os.path.join(HERE, f"det_{tag}_320.npz"), head=head.numpy(), dets=aware.numpy(), dets_agnostic=agnostic.numpy(),
                            conf=AWARE[0], nms=AWARE[1], conf_agnostic=AGNOSTIC[0], nms_agnostic=AGNOSTIC[1], seed_video=1, n_obj=3, frame=1)


if __name__ == "__main__":
    main()

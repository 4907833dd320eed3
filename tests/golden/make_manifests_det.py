"""Dump the state_dict key->shape manifests of the COCO detectors (exps/default/unicorn_det_*_800x1280.py) from the reference (build
container only), like make_manifests.py does for the tracking configs.  They pin unicorn_b200.weights.param_shapes() for
unicorn_det_convnext_tiny / unicorn_det_convnext_large / unicorn_det_r50."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle"))
sys.path.insert(0, HERE)
import ref_import  # noqa: E402
from make_golden_r50 import install_offline_resnet  # noqa: E402

install_offline_resnet()
for name in ("unicorn_det_convnext_tiny", "unicorn_det_convnext_large", "unicorn_det_r50"):
    _, m = ref_import.get_model(name + "_800x1280")
    sd = m.state_dict()
    man = {k: list(v.shape) for k, v in sd.items()}
    with open(os.path.join(HERE, f"manifest_{name}.json"), "w") as f:
        json.dump(man, f, indent=0, sort_keys=False)
    print(name, len(man), sum(v.numel() for v in sd.values()) / 1e6, "M")

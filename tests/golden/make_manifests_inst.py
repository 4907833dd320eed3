"""Dump the state_dict key->shape manifest of the COCO instance segmenter (exps/default/unicorn_inst_convnext_tiny_800x1280.py) from
the reference (build container only), like make_manifests_det.py does for the detectors.  It pins
unicorn_b200.weights.param_shapes("unicorn_inst_convnext_tiny")."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle"))
import ref_import  # noqa: E402

name = "unicorn_inst_convnext_tiny"
_, m = ref_import.get_model(name + "_800x1280")
sd = m.state_dict()
man = {k: list(v.shape) for k, v in sd.items()}
with open(os.path.join(HERE, f"manifest_{name}.json"), "w") as f:
    json.dump(man, f, indent=0, sort_keys=False)
print(name, len(man), sum(v.numel() for v in sd.values()) / 1e6, "M")

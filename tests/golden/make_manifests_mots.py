"""Dump the state_dict key->shape manifest of the MOTS Challenge model from the reference (build container only), like
make_manifests.py does for the other ConvNeXt configs.  It pins unicorn_b200.weights.param_shapes() for
unicorn_track_large_mot_challenge_mask."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle"))
import ref_import  # noqa: E402

for name in ("unicorn_track_large_mot_challenge_mask",):
    _, m = ref_import.get_model(name)
    sd = m.state_dict()
    man = {k: list(v.shape) for k, v in sd.items()}
    with open(os.path.join(HERE, f"manifest_{name}.json"), "w") as f:
        json.dump(man, f, indent=0, sort_keys=False)
    print(name, len(man), sum(v.numel() for v in sd.values()) / 1e6, "M")

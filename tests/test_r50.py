"""ResNet-50 tracking configs (unicorn_track_r50, unicorn_track_r50_mask) without a GPU: parameter table, BatchNorm folding,
checkpoint validation and the drop-in Exp."""
import os
import subprocess
import sys
import textwrap

import pytest
import torch
import torch.nn.functional as F

from unicorn_b200.weights import CONFIGS, fold_bn, load_checkpoint, make_state_dict, param_shapes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R50 = ("unicorn_track_r50", "unicorn_track_r50_mask")


def test_r50_param_counts():
    n = lambda name: sum(int(torch.tensor(s).prod()) for s in param_shapes(name).values())  # noqa: E731
    # the reference's state_dicts: 666 / 701 tensors (the 53 int64 num_batches_tracked scalars count one element each)
    assert len(param_shapes("unicorn_track_r50")) == 666 and len(param_shapes("unicorn_track_r50_mask")) == 701
    assert n("unicorn_track_r50") == 122979950
    assert n("unicorn_track_r50_mask") == 129036167
    bb = [k for k in param_shapes("unicorn_track_r50") if k.startswith("backbone.backbone.") and k.endswith("running_var")]
    assert len(bb) == 53


def test_in_channels():
    assert CONFIGS["unicorn_track_r50"]["in_channels"] == (512, 1024, 2048)
    assert CONFIGS["unicorn_track_large"]["in_channels"] == (384, 768, 1536)
    assert CONFIGS["unicorn_track_tiny_mask"]["in_channels"] == (192, 384, 768)
    s = param_shapes("unicorn_track_r50_mask")
    assert s["bottleneck.0.weight"] == (256, 1024, 1, 1) and s["head.stems.2.conv.weight"] == (256, 2048, 1, 1)
    assert s["head.mask_branch.refine.0.0.weight"] == (128, 512, 3, 3) and s["backbone.lateral_conv0.conv.weight"] == (1024, 2048, 1, 1)


@pytest.mark.parametrize("k,stride", [(1, 1), (3, 2), (1, 2), (7, 2)])
def test_fold_bn_equals_conv_then_eval_batchnorm(k, stride):
    g = torch.Generator().manual_seed(k * 10 + stride)
    w = torch.randn(32, 16, k, k, generator=g, dtype=torch.float64)
    sd = {"bn.weight": torch.randn(32, generator=g), "bn.bias": torch.randn(32, generator=g),
          "bn.running_mean": torch.randn(32, generator=g), "bn.running_var": torch.rand(32, generator=g) + 0.01}
    x = torch.randn(2, 16, 23, 19, generator=g, dtype=torch.float64)
    ref = F.batch_norm(F.conv2d(x, w, stride=stride, padding=k // 2), sd["bn.running_mean"].double(), sd["bn.running_var"].double(),
                       sd["bn.weight"].double(), sd["bn.bias"].double(), False, 0.0, 1e-3)
    wf, bf = fold_bn(w, sd, "bn.")
    got = F.conv2d(x, wf, bf, stride=stride, padding=k // 2)
    assert wf.dtype == torch.float64 and (got - ref).abs().max().item() < 1e-12 * ref.abs().max().item() + 1e-12


def test_seeded_r50_weights_are_well_conditioned():
    sd = make_state_dict("unicorn_track_r50", 0)
    nbt = [k for k in sd if k.endswith("num_batches_tracked")]
    assert len(nbt) == 53 and all(sd[k].dtype == torch.int64 and sd[k].dim() == 0 for k in nbt)
    assert all((sd[k] > 0).all() for k in sd if k.endswith("running_var"))
    assert all(sd[k].abs().mean() < 0.5 for k in sd if k.endswith("bn3.weight"))
    # the ConvNeXt configs are untouched by the R50 rules
    assert not any("running" in k for k in make_state_dict("unicorn_track_tiny", 0))


def test_r50_features_stay_o1():
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import resnet_oracle as ro
    sd = make_state_dict("unicorn_track_r50", 0)
    img = torch.rand(1, 3, 128, 128, generator=torch.Generator().manual_seed(0)) * 255
    with torch.no_grad():
        feats = ro.resnet50_features(img, sd, ro.CONFIGS["unicorn_track_r50"])
    assert [f.shape[1] for f in feats] == [512, 1024, 2048]
    assert all(0.05 < f.std().item() and f.abs().max().item() < 50 for f in feats)


@pytest.mark.parametrize("name", R50)
def test_load_checkpoint_accepts_released_r50_layout(tmp_path, name):
    sd = make_state_dict(name, 0)
    p = tmp_path / "best_ckpt.pth"
    torch.save({"model": {k: (v.half() if v.is_floating_point() else v) for k, v in sd.items()}, "start_epoch": 3}, p)
    got = load_checkpoint(str(p), name)
    assert list(got) == list(sd)
    k = "backbone.backbone.layer1.0.bn1.num_batches_tracked"
    assert got[k].dtype == torch.int64 and got[k].dim() == 0
    assert got["backbone.backbone.bn1.running_var"].dtype == torch.float32
    bad = dict(sd)
    del bad["backbone.backbone.layer3.2.bn2.running_mean"]
    with pytest.raises(ValueError, match="does not match"):
        load_checkpoint(bad, name)


def test_shim_get_exp_r50():
    code = textwrap.dedent(f"""
        import sys
        sys.path.insert(0, {ROOT!r})
        import unicorn_b200.shim as shim
        shim.install()
        from unicorn.exp import get_exp
        for name in {R50!r}:
            exp = get_exp(f"exps/default/{{name}}.py", None)
            assert exp.backbone_name == "resnet50" and exp.in_channels == [512, 1024, 2048], (exp.backbone_name, exp.in_channels)
            assert exp.mask == name.endswith("_mask") and exp.num_classes == 8
        exp = get_exp("exps/default/unicorn_track_large.py", None)
        assert exp.backbone_name == "convnext_large" and exp.in_channels == [384, 768, 1536]
        print("r50 exp ok")
    """)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "r50 exp ok" in r.stdout, r.stdout + r.stderr


def _rel(a, b):
    a, b = torch.as_tensor(a).float(), torch.as_tensor(b).float()
    return ((a - b).abs().max() / (b.abs().max() + 1e-12)).item()


def test_oracle_r50_sot_matches_reference_golden():
    """oracle SOT frames of unicorn_track_r50 against tests/golden/sot_r50_320.npz (UNMODIFIED reference,
    tests/golden/make_golden_r50.py)."""
    import numpy as np
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import resnet_oracle as ro
    from unicorn_b200.synthetic import make_video
    g = np.load(os.path.join(ROOT, "tests", "golden", "sot_r50_320.npz"))
    name, nf = str(g["config"]), int(g["n_frames"])
    sd = make_state_dict(name, 0)
    frames, boxes = make_video(nf, 320, 320, seed=int(g["seed"]))
    o = ro.SOTOracle(sd, name)
    o.initialize(frames[0:1], boxes[0, 0])
    st = {}
    with torch.no_grad():
        for t in range(1, nf):
            o.track(frames[t:t + 1], st)
        x2, x1, x0 = ro.resnet50_features(frames[nf - 1:nf], sd, ro.CONFIGS[name])
    assert _rel(x2[0, ::8, ::2, ::2], g["x2_sub"]) < 1e-4 and _rel(x1[0, ::8], g["x1_sub"]) < 1e-4 and _rel(x0[0, ::16], g["x0_sub"]) < 1e-4
    assert _rel(st["fpn"][1][0, ::4], g["fpn1_sub"]) < 1e-4 and _rel(st["feat"][0, ::8], g["feat_sub"]) < 1e-4
    assert _rel(st["coarse"], g["coarse"]) < 1e-4 and _rel(st["head"], g["head"]) < 1e-4
    ref = torch.from_numpy(g["dets"])
    assert st["dets"].shape == ref.shape
    assert torch.cdist(st["dets"][:, :6], ref[:, :6], p=float("inf")).min(dim=0)[0].max().item() / ref[:, :6].abs().max().item() < 1e-4


def test_oracle_r50_mask_whole_matches_reference_golden():
    import numpy as np
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import resnet_oracle as ro
    import unicorn_oracle as orc
    from unicorn_b200.synthetic import make_video
    g = np.load(os.path.join(ROOT, "tests", "golden", "whole_r50_mask_320.npz"))
    name = str(g["config"])
    frames, _ = make_video(2, 320, 320, seed=int(g["seed_video"]), n_obj=int(g["n_obj"]))
    img = frames[int(g["frame"]):int(g["frame"]) + 1]
    with torch.no_grad():
        (outs, locs, dyn, lvls, mf, um), seq = ro.whole_forward(img, make_state_dict(name, 0), ro.CONFIGS[name])
    assert outs.shape == (1, 2100, 13) and _rel(outs, g["head"]) < 1e-4 and _rel(dyn[0, ::16], g["dyn_sub"]) < 1e-4
    assert _rel(mf, g["mask_feats"]) < 1e-4 and _rel(um[0, :, ::4, ::4], g["up_masks_sub"]) < 1e-4
    assert _rel(seq["feat"][0, ::8], g["feat_sub"]) < 1e-4
    dets = orc.postprocess(outs, 8, float(g["conf"]), float(g["nms"]))[0]
    ref = torch.from_numpy(g["dets"])
    assert dets.shape == ref.shape
    assert torch.cdist(dets[:, :6], ref[:, :6], p=float("inf")).min(dim=0)[0].max().item() / ref[:, :6].abs().max().item() < 1e-4

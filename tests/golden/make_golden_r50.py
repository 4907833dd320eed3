"""Golden fixtures of the ResNet-50 tracking models from the UNMODIFIED reference (build container only), with the oracle checked
against them (< 1e-4 relative):

  sot_r50_320.npz         unicorn_track_r50: SOT frames following external/lib/test/tracker/unicorn_sot.py:39-109 (fp32 correlation),
                          as tests/golden/make_golden.py does for the tiny model: backbone outputs, feat, prior, head and detections.
  whole_r50_mask_320.npz  unicorn_track_r50_mask: `mode="whole"` (unicorn.py:133-139) UnicornHeadMask outputs, dynamic parameters,
                          mask features and postprocess detections, as tests/golden/make_golden_whole.py does for the tiny mask model.

    python tests/golden/make_golden_r50.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, HERE)
import ref_import  # noqa: E402
import resnet_oracle as ro  # noqa: E402
import unicorn_oracle as orc  # noqa: E402
from make_golden import maxrel, run_reference_sot  # noqa: E402
from unicorn_b200.synthetic import make_video  # noqa: E402
from unicorn_b200.weights import make_state_dict  # noqa: E402

H = W = 320


def install_offline_resnet():
    """ref_import.install(), then stub the ImageNet download of resnet50(pretrained=True) (backbone/yolo_pafpn_new.py:45-46,
    backbone/resnet.py:230-236): offline the backbone keeps its initialisation, and the state_dict loaded afterwards replaces it."""
    ref_import.install()
    import unicorn.models.backbone.resnet as rn
    rn.load_state_dict_from_url = lambda *a, **k: {}


install_offline_resnet()
CONF, NMS = 0.01, 0.7  # whole mode: the track_omni CLI thresholds (tools/track_omni.py:100-101)


def sot():
    name, nf = "unicorn_track_r50", 3
    sd = make_state_dict(name, seed=0)
    _, model = ref_import.get_model(name)
    print(model.load_state_dict(sd, strict=True))
    frames, boxes = make_video(nf, H, W, seed=0)
    ref = run_reference_sot(model, frames, boxes[0, 0])
    o = ro.SOTOracle(sd, name)
    o.initialize(frames[0:1], boxes[0, 0])
    worst = 0.0
    for t in range(1, nf):
        st = {}
        o.track(frames[t:t + 1], st)
        r = ref[t - 1]
        for k in ("feat", "inter_cur", "embed_cur", "coarse", "head"):
            e = maxrel(st[k], r[k]); worst = max(worst, e)
            print(f"frame {t} {k:10s} oracle-vs-reference max rel err {e:.3e}")
        for i in range(3):
            e = maxrel(st["fpn"][i], r["fpn"][i]); worst = max(worst, e)
        assert st["dets"].shape == r["dets"].shape, (st["dets"].shape, r["dets"].shape)
        d = torch.cdist(st["dets"][:, :6], r["dets"][:, :6], p=float("inf")).min(dim=0)[0].max().item() / r["dets"][:, :6].abs().max().item()
        worst = max(worst, d)
    assert worst < 1e-4, worst
    # the backbone outputs themselves (the reference's model.backbone.backbone on the last frame)
    with torch.no_grad():
        x2, x1, x0 = model.backbone.backbone(frames[nf - 1:nf])
    o_feats = ro.resnet50_features(frames[nf - 1:nf], sd, ro.CONFIGS[name])
    for a, b in zip(o_feats, (x2, x1, x0)):
        e = maxrel(a, b)
        print("resnet50 output oracle-vs-reference", tuple(b.shape), f"{e:.3e}")
        assert e < 1e-4
    r = ref[-1]
    np.savez_compressed(os.path.join(HERE, "sot_r50_320.npz"), config=name, seed=0, n_frames=nf, H=H, W=W, init_box=boxes[0, 0].numpy(),
                        x2_sub=x2[0, ::8, ::2, ::2].numpy(), x1_sub=x1[0, ::8].numpy(), x0_sub=x0[0, ::16].numpy(),
                        fpn1_sub=r["fpn"][1][0, ::4].numpy(), feat_sub=r["feat"][0, ::8].numpy(), coarse=r["coarse"].numpy(),
                        head=r["head"].numpy(), dets=r["dets"].numpy())
    print("wrote sot_r50_320.npz; worst oracle-vs-reference rel err", worst)


def whole_mask():
    name = "unicorn_track_r50_mask"
    sd = make_state_dict(name, 0)
    _, model = ref_import.get_model(name)
    print(model.load_state_dict(sd, strict=True))
    from unicorn.utils.boxes import postprocess
    frames, _ = make_video(2, H, W, seed=1, n_obj=3)
    img = frames[1:2]
    with torch.no_grad():
        (outs, locs, dyn, lvls, mf, um), seq = model(img, mode="whole")
        dets = postprocess(outs.clone(), 8, CONF, NMS)[0]
        o = ro.whole_forward(img, sd, ro.CONFIGS[name])[0]
    for a, b, n in zip(o, (outs, locs, dyn, lvls, mf, um), ("outputs", "locations", "dyn", "levels", "mask_feats", "up_masks")):
        e = maxrel(a.float(), b.float())
        print(f"r50 mask whole {n:10s} oracle-vs-reference rel err {e:.3e}")
        assert e < 1e-4
    o_dets = orc.postprocess(o[0], 8, CONF, NMS)[0]
    assert o_dets.shape == dets.shape, (o_dets.shape, dets.shape)
    d = torch.cdist(o_dets[:, :6], dets[:, :6], p=float("inf")).min(dim=0)[0].max().item() / dets[:, :6].abs().max().item()
    assert d < 1e-4, d
    np.savez_compressed(os.path.join(HERE, "whole_r50_mask_320.npz"), config=name, conf=CONF, nms=NMS, seed_video=1, n_obj=3, frame=1,
                        head=outs.numpy(), dyn_sub=dyn[0, ::16].numpy(), mask_feats=mf.numpy(), up_masks_sub=um[0, :, ::4, ::4].numpy(),
                        dets=dets.numpy(), feat_sub=seq["feat"][0, ::8].numpy())
    print("wrote whole_r50_mask_320.npz")


if __name__ == "__main__":
    sot()
    whole_mask()

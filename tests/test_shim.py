"""The `unicorn`-importable shim (unicorn_b200/shim): API surface on CPU, stopping with this package's loud no-fallback error
where the GPU is needed (`.cuda()`)."""
import os
import subprocess
import sys
import textwrap

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_shim_surface():
    code = textwrap.dedent(f"""
        import sys
        sys.path.insert(0, {ROOT!r})
        import unicorn_b200.shim as shim
        shim.install()
        import torch
        from unicorn.exp import get_exp, ExpTrack
        from unicorn.utils import postprocess, fuse_model
        from unicorn.utils.boxes import postprocess_inst
        from unicorn.tracker.byte_tracker import BYTETracker, STrack
        from unicorn.tracker.quasi_dense_embed_tracker import QuasiDenseEmbedTracker
        from unicorn.models import Unicorn
        from unicorn_b200.weights import make_state_dict
        from unicorn_b200._lib import UnicornB200Error
        exp = get_exp("exps/default/unicorn_track_tiny_mask.py", None)
        assert exp.test_size == (800, 1280) and exp.normalize is False and exp.d_rate == 2 and exp.use_raft and exp.num_classes == 8
        exp.merge(["test_conf", "0.01"]); assert exp.test_conf == 0.01
        model = exp.get_model(load_pretrain=False)
        assert isinstance(model, Unicorn) and model.head.mask_head is not None and model.head.decode_in_inference
        sd = make_state_dict("unicorn_track_tiny_mask", 0)
        sd["head.mask_head._iter"] = torch.zeros(1)          # a buffer of the reference's DynamicMaskHead: tolerated
        r = model.load_state_dict(sd, strict=True)
        assert not r.missing_keys
        bad = dict(sd); bad.pop("head.stems.0.conv.weight")
        for strict in (True, False):
            try:
                model.load_state_dict(bad, strict=strict); raise SystemExit("missing key accepted")
            except RuntimeError:
                pass
        assert model.eval() is model and model.half() is model
        try:
            model(imgs=torch.zeros(1, 3, 32, 32), mode="backbone"); raise SystemExit("ran without a GPU engine")
        except RuntimeError:
            pass
        if not torch.cuda.is_available():
            try:
                model.cuda(); raise SystemExit("built an engine without a GPU")
            except UnicornB200Error:
                pass
        try:
            get_exp("exps/default/yolox_s.py", None); raise SystemExit("unknown config accepted")
        except KeyError:
            pass
        print("shim surface ok")
    """)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "shim surface ok" in r.stdout, r.stdout + r.stderr


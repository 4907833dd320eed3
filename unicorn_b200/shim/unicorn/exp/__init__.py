"""unicorn.exp — get_exp / Exp for the tracking configs of the per-frame path (reference: unicorn/exp/build.py:35-50,
unicorn/exp/unicorn_track.py:30-122, unicorn_track_mask.py:31-46, exps/default/unicorn_track_*.py).

get_exp(exp_file, exp_name) keeps the reference's signature: the config is identified by the file's base name (the file itself is
not executed — the reference's Exp classes build PyTorch training objects that do not exist here)."""
import os

from unicorn_b200.compat.model import UnicornB200Model
from unicorn_b200.weights import CONFIGS


class Exp:
    """Attributes read by the inference drivers (unicorn_sot.py:18-25, unicorn_vos.py:19-31, tools/track_omni.py:150-201)."""

    def __init__(self, exp_name):
        if exp_name not in CONFIGS:
            raise KeyError(f"unicorn_b200 has no config {exp_name!r} (known: {sorted(CONFIGS)})")
        cfg = CONFIGS[exp_name]
        self.exp_name = exp_name
        if cfg["task"] == "det":
            self._init_det(cfg)
            return
        self.num_classes = cfg["num_classes"]       # unicorn_track.py:36 (8) / *_mot_challenge.py:18 (1)
        if cfg["backbone"] == "resnet50":
            self.backbone_name = "resnet50"          # exps/default/unicorn_track_r50*.py
        else:
            self.backbone_name = "convnext_tiny" if "tiny" in exp_name else "convnext_large"
        self.in_channels = list(cfg["in_channels"])  # unicorn_track.py:43, exps/default/unicorn_track_large.py:15, *_r50*.py
        self.normalize = False                      # unicorn_track.py:76
        self.test_size = (800, 1280)                # unicorn_track.py:104
        self.input_size = (800, 1280)
        self.test_conf = 0.001                      # unicorn_track.py (YOLOX default)
        self.nmsthre = 0.65
        self.grid_sample = False
        self.output_dir = "./Unicorn_outputs"
        self.mask = cfg["mask"]
        if cfg["mask"]:
            self.use_raft = True                    # unicorn_track_mask.py:44
            self.d_rate = 2                         # unicorn_track_mask.py:45
            self.ctrl_loc = "reg"                   # unicorn_track_mask.py:38
        self.model = None

    def _init_det(self, cfg):
        """exp/unicorn_det.py:22-92 with exps/default/unicorn_det_*_800x1280.py: the COCO detector (YOLOX + YOLOXHeadDet); with
        exp/unicorn_det_mask.py (exps/default/unicorn_inst_convnext_tiny_800x1280.py) the instance segmenter (YOLOXHeadDetMask)."""
        self.task = "det"
        self.num_classes = cfg["num_classes"]      # unicorn_det.py:25 (COCO)
        if cfg["backbone"] == "resnet50":
            self.backbone_name = "resnet50"         # unicorn_det_r50_800x1280.py
        else:
            self.backbone_name = "convnext_large" if "large" in self.exp_name else "convnext"  # unicorn_det.py:30
        self.in_channels = list(cfg["in_channels"])
        self.normalize = False                     # unicorn_det.py:62
        self.test_size = (800, 1280)               # exps/default/unicorn_det_*_800x1280.py
        self.input_size = (800, 1280)
        self.test_conf = 0.01                      # unicorn_det.py:88-89
        self.nmsthre = 0.65
        self.output_dir = "./Unicorn_outputs"
        self.mask_thres = 0.3                      # unicorn_det.py:92
        self.mask = cfg["mask"]
        if cfg["mask"]:                            # exp/unicorn_det_mask.py:22-44 (ExpDetMask): CondInst with the RAFT upsampler
            self.task = "inst"
            self.ctrl_loc = "reg"
            self.use_raft = True
            self.d_rate = 2
            self.sem_loss_on = False
        self.model = None

    def get_model(self, load_pretrain=True):
        """exp/unicorn_track.py:115-193.  Returns the H100 model shell; weights come from load_state_dict (there is no
        Unicorn_outputs/<pretrain>/best_ckpt.pth lookup: pass load_pretrain=False like the reference's inference drivers)."""
        if load_pretrain:
            raise RuntimeError("get_model(load_pretrain=True) would read a COCO-pretrained checkpoint for training; the inference "
                               "drivers call get_model(load_pretrain=False) and load_state_dict the tracking checkpoint")
        if self.model is None:
            self.model = UnicornB200Model(None, self.exp_name)
        return self.model

    def merge(self, cfg_list):
        assert len(cfg_list) % 2 == 0
        for k, v in zip(cfg_list[0::2], cfg_list[1::2]):
            if hasattr(self, k):
                src = getattr(self, k)
                if src is not None and not isinstance(v, type(src)):
                    try:
                        v = type(src)(v)
                    except Exception:
                        import ast
                        v = ast.literal_eval(v)
                setattr(self, k, v)


ExpTrack = ExpTrackMask = ExpDet = ExpDetMask = Exp


def get_exp(exp_file=None, exp_name=None):
    """unicorn/exp/build.py:35-50."""
    assert exp_file is not None or exp_name is not None, "plz provide exp file or exp name."
    name = os.path.basename(exp_file).split(".")[0] if exp_file is not None else exp_name
    # exps/default/unicorn_det_*_800x1280.py and unicorn_inst_*_800x1280.py: the input size is an attribute of the Exp, not part of the config
    if name.startswith(("unicorn_det_", "unicorn_inst_")) and name.endswith("_800x1280"):
        name = name[:-len("_800x1280")]
    return Exp(name)

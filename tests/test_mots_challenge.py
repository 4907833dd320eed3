"""The MOTS Challenge model (unicorn_track_large_mot_challenge_mask: ConvNeXt-L, one class, mask head) on the CPU side, and the argument
checks of uc_mots_encode, which come before any CUDA call."""
import ctypes
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "unicorn_track_large_mot_challenge_mask"


def test_get_exp_serves_the_mots_challenge_model():
    from unicorn_b200.shim.unicorn.exp import get_exp
    exp = get_exp(f"exps/default/{NAME}.py", None)
    assert exp.num_classes == 1 and exp.mask and exp.use_raft and exp.d_rate == 2
    assert exp.backbone_name == "convnext_large" and exp.in_channels == [384, 768, 1536]


def test_oracle_builds_the_mots_challenge_model():
    """The oracle runs the combination: the 1-class head of *_mot_challenge with the mask head of *_mask."""
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import unicorn_oracle as orc
    from unicorn_b200.weights import make_state_dict
    cfg = dict(orc.CONFIGS["unicorn_track_large_mot_challenge"], mask=True)
    img = torch.rand(1, 3, 64, 64, generator=torch.Generator().manual_seed(0)) * 255
    with torch.no_grad():
        (outs, locs, dyn, lvls, mf, um), _ = orc.whole_forward(img, make_state_dict(NAME, 0), cfg)
    A = 8 * 8 + 4 * 4 + 2 * 2
    assert outs.shape == (1, A, 6) and dyn.shape == (1, A, 169) and mf.shape == (1, 8, 8, 8) and um.shape == (1, 144, 8, 8)
    assert torch.isfinite(outs).all() and torch.isfinite(mf).all()


def test_mots_encode_validates_arguments_before_any_launch():
    from unicorn_b200 import _lib
    lib = _lib.lib()
    lib.uc_last_error.restype = ctypes.c_char_p
    lib.uc_mots_encode_workspace_bytes.restype = ctypes.c_long
    P, D, L = ctypes.c_void_p, ctypes.c_double, ctypes.c_long
    m, o, e, ws, ch, off = P(0x10000), P(0x20000), P(0x30000), P(0x40000), P(0x50000), P(0x60000)  # never dereferenced
    need = lib.uc_mots_encode_workspace_bytes(4, 1080, 1920)
    assert need > 0 and lib.uc_mots_encode_workspace_bytes(-1, 1080, 1920) < 0

    def call(masks=m, n_max=8, Hin=800, Win=1280, order=o, emit=e, k=4, r=0.75, H=1080, W=1920, work=ws, wbytes=need, chars=ch,
             cap=1000, offsets=off):
        rc = lib.uc_mots_encode(masks, n_max, Hin, Win, order, emit, k, ctypes.c_float(0.3), D(r), H, W, work, L(wbytes), chars, L(cap),
                                offsets, None)
        return rc, lib.uc_last_error()

    for kw in (dict(masks=None), dict(order=None), dict(emit=None), dict(offsets=None), dict(work=None), dict(chars=None)):
        assert call(**kw) == (-1, b"uc_mots_encode: null pointer"), kw
    for kw in (dict(n_max=0), dict(Hin=0), dict(Win=-3), dict(H=0), dict(W=0), dict(r=0.0), dict(r=-1.0)):
        rc, msg = call(**kw)
        assert rc == -1 and b"bad sizes" in msg, kw
    assert call(k=9)[0] == -1 and b"must be in 0..n_max" in call(k=9)[1]
    assert call(k=-1)[0] == -1 and b"must be in 0..n_max" in call(k=-1)[1]
    assert call(cap=-1)[0] == -1 and b"negative capacity" in call(cap=-1)[1]
    for kw in (dict(masks=P(0x10002)), dict(order=P(0x20001)), dict(offsets=P(0x60004)), dict(work=P(0x40008))):
        rc, msg = call(**kw)
        assert rc == -1 and b"aligned" in msg, kw
    assert call(wbytes=16)[0] == -1 and b"workspace too small" in call(wbytes=16)[1]
    assert call(r=1e4)[0] == -1 and b"empty" in call(r=1e4)[1]

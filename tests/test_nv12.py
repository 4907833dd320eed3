"""NV12 frames without a GPU: the numpy restatement of the NV12 letterbox is pinned bit for bit to the reference path for an NV12
frame (cv2.cvtColor(COLOR_YUV2RGB_NV12), then the SOT preprocessor), malformed 2-D frames are rejected, and uc_letterbox_nv12
rejects every bad argument with UC_EINVAL before anything is launched (fake addresses, never dereferenced)."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

from unicorn_b200 import _lib
from unicorn_b200.sot import nv12_size, preprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
SOURCES = [(2, 2), (480, 640), (720, 1280), (1080, 1920), (362, 498), (320, 320), (800, 1280)]  # the last two fit one target exactly
TARGETS = [(800, 1280), (320, 320)]


def nv12_frame(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h * 3 // 2, w), dtype=np.uint8)


@pytest.mark.parametrize("size", TARGETS)
@pytest.mark.parametrize("hw", SOURCES)
def test_oracle_equals_cv2_recipe(hw, size):
    cv2 = pytest.importorskip("cv2")
    import nv12_oracle
    nv12 = nv12_frame(*hw, seed=hw[0] * 7 + hw[1])
    ref, r = preprocess(cv2.cvtColor(nv12, cv2.COLOR_YUV2RGB_NV12), size, out=torch.empty(1, *size, 3, dtype=torch.uint8))
    out, r2 = nv12_oracle.letterbox_nv12(nv12, size)
    assert r2 == r
    assert np.array_equal(out, ref[0].numpy())


def test_oracle_conversion_equals_cv2_on_every_chroma_pair():
    """Every (U, V) pair of a 256 x 256 chroma lattice, each under a 2 x 2 block of random luma, converts as cv2 converts it."""
    cv2 = pytest.importorskip("cv2")
    import nv12_oracle
    h, w = 512, 512
    nv12 = nv12_frame(h, w, seed=5)
    uv = nv12[h:].reshape(h // 2, w // 2, 2)
    uv[..., 0] = np.arange(256, dtype=np.uint8)[:, None]
    uv[..., 1] = np.arange(256, dtype=np.uint8)[None, :]
    assert np.array_equal(nv12_oracle.nv12_to_bgr(nv12), cv2.cvtColor(nv12, cv2.COLOR_YUV2BGR_NV12))


@pytest.mark.parametrize("shape,dtype", [((5, 4), np.uint8), ((6, 3), np.uint8), ((6, 4), np.float32), ((0, 4), np.uint8),
                                         ((6, 0), np.uint8)])
def test_malformed_2d_frames_are_rejected(shape, dtype):
    """Rows not a multiple of 3, odd w, a non-uint8 array, an empty frame: ValueError, for numpy arrays and tensors alike (with
    rows a multiple of 3, h = 2 rows / 3 is even)."""
    a = np.zeros(shape, dtype=dtype)
    for frame in (a, torch.from_numpy(a)):
        with pytest.raises(ValueError, match="NV12"):
            nv12_size(frame)


def test_nv12_size():
    assert nv12_size(np.zeros((1620, 1920), np.uint8)) == (1080, 1920)
    assert nv12_size(torch.zeros(3, 2, dtype=torch.uint8)) == (2, 2)
    assert nv12_size(np.zeros((12, 16), np.uint8)[:, 2:10]) == (8, 8)  # a view of a wider buffer
    assert nv12_size(np.zeros((4, 6, 3), np.uint8)) is None  # an RGB frame is left to the path that reads it
    assert nv12_size(np.zeros((4, 6, 2), np.uint8)) is None


P = ctypes.c_void_p
Y, UV, DST = P(0x10000), P(0x20000), P(0x30000)  # never dereferenced


def nv12_call(y=Y, uv=UV, ld=64, Hs=48, Ws=64, dst=DST, Hd=32, Wd=32, rh=24, rw=32, pad=114):
    lib = _lib.lib()
    return lib.uc_letterbox_nv12(y, uv, ld, Hs, Ws, dst, Hd, Wd, rh, rw, pad, None), lib.uc_last_error()


@pytest.mark.parametrize("kw,words", [
    (dict(y=None), "null plane"), (dict(uv=None), "null plane"), (dict(dst=None), "destination"),
    (dict(Hs=47), "even"), (dict(Ws=63, ld=64), "even"), (dict(Hs=0), "even"), (dict(Ws=0), "even"),
    (dict(ld=62), "ld must be >= Ws"),
    (dict(rh=0), "rh, rw"), (dict(rw=0), "rh, rw"), (dict(rh=33), "rh, rw"), (dict(rw=33), "rh, rw"), (dict(Hd=0, rh=1), "rh, rw"),
    (dict(pad=-1), "pad"), (dict(pad=256), "pad")])
def test_letterbox_nv12_rejects_bad_arguments(kw, words):
    rc, msg = nv12_call(**kw)
    assert rc == -1, (rc, msg)  # UC_EINVAL
    assert b"uc_letterbox_nv12" in msg and words.encode() in msg, msg


@pytest.mark.parametrize("src", [np.zeros((6, 4), np.uint8), torch.zeros(6, 4, 3, dtype=torch.uint8), torch.zeros(5, 4, dtype=torch.uint8),
                                 torch.zeros(6, 4, dtype=torch.int16), torch.zeros(6, 8, dtype=torch.uint8)[:, ::2],
                                 torch.zeros(1, 4, dtype=torch.uint8).expand(6, 4), torch.zeros(6, 4, dtype=torch.uint8)])
def test_letterbox_nv12_wrapper_rejects_bad_sources(src):
    """A numpy array, a 3-D or 5-row tensor, a non-uint8 tensor, a non-unit column stride, a row stride below w, a host tensor:
    ValueError before anything reaches the device."""
    from unicorn_b200 import shared_ops
    with pytest.raises(ValueError, match="letterbox_nv12"):
        shared_ops.letterbox_nv12(src, (32, 32))

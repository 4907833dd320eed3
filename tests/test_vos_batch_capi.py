"""The batched mask entry points (uc_aligned_bilinear_add_batched, uc_dynamic_masks_batched) reject a bad image count, null pointers
and per-image strides smaller than one image with UC_EINVAL and a message prefixed by the entry point's name, before any CUDA call
(so this runs without a GPU)."""
import ctypes

import pytest

P = ctypes.c_void_p
L = ctypes.c_long
A_, B_, C_, D_, E_, F_ = (P(0x100000 * k) for k in range(1, 7))  # never dereferenced: validation comes first


@pytest.fixture(scope="module")
def lib():
    from unicorn_b200 import _lib
    lib = _lib.lib()
    lib.uc_last_error.restype = ctypes.c_char_p
    return lib


def err(lib, rc, prefix):
    assert rc == -1, rc
    msg = lib.uc_last_error()
    assert msg.startswith(prefix + b":"), msg
    return msg


def ab(lib, B, src=A_, dst=B_, bs_src=20 * 30 * 128, bs_dst=40 * 60 * 128):
    # 20 x 30 source pixels of 128 channels, factor 2
    return lib.uc_aligned_bilinear_add_batched(src, 128, L(bs_src), 20, 30, dst, 128, L(bs_dst), 128, 2, B, None)


def test_aligned_bilinear_add_batched_rejects_bad_arguments(lib):
    name = b"uc_aligned_bilinear_add_batched"
    for B in (0, -1):
        assert b"B must be >= 1" in err(lib, ab(lib, B), name)
    assert b"null pointer" in err(lib, ab(lib, 2, src=None), name)
    assert b"null pointer" in err(lib, ab(lib, 2, dst=None), name)
    for kw in (dict(bs_src=20 * 30 * 128 - 2), dict(bs_dst=40 * 60 * 128 - 2), dict(bs_src=20 * 30 * 128 + 1)):
        assert b"bad per-image strides" in err(lib, ab(lib, 3, **kw), name), kw


def dm(lib, B, S=2, bs_dyn=(100 * 176, 25 * 176, 4 * 176), bs_anchors=129, image_of=F_, mask_feats=A_, anchors=D_, count=E_):
    # h x w = 10 x 10 mask map; levels 10x10, 5x5, 2x2 (129 anchors); n_max 1; up 4, d 2
    dyn = (P * 3)(C_, C_, C_)
    hw = (ctypes.c_int * 6)(10, 10, 5, 5, 2, 2)
    st = (ctypes.c_int * 3)(8, 16, 32)
    so = (ctypes.c_float * 3)(64.0, 128.0, 256.0)
    bs = (L * 3)(*bs_dyn) if bs_dyn is not None else None
    return lib.uc_dynamic_masks_batched(mask_feats, B_, S, 10, 10, 4, 2, dyn, 176, bs, hw, st, so, anchors, L(bs_anchors), count, image_of, B, 1,
                                        C_, D_, None)


def test_dynamic_masks_batched_rejects_bad_arguments(lib):
    name = b"uc_dynamic_masks_batched"
    for B in (0, -3):
        assert b"B must be >= 1" in err(lib, dm(lib, B), name)
    assert b"S (mask-branch images) must be >= 1" in err(lib, dm(lib, 2, S=0), name)
    for kw in (dict(mask_feats=None), dict(anchors=None), dict(count=None)):
        assert b"null pointer" in err(lib, dm(lib, 2, **kw), name), kw
    assert b"image_of" in err(lib, dm(lib, 2, image_of=None), name)
    assert b"null pointer" in err(lib, dm(lib, 2, bs_dyn=None), name)
    msg = err(lib, dm(lib, 2, bs_dyn=(100 * 176, 25 * 176 - 1, 4 * 176)), name)
    assert b"bad per-image strides of level 1" in msg
    assert b"bad per-image strides of level 2" in err(lib, dm(lib, 2, bs_dyn=(100 * 176, 25 * 176, 0)), name)
    assert b"anchor stride" in err(lib, dm(lib, 2, bs_anchors=128), name)


def test_unbatched_entry_points_keep_their_messages(lib):
    """The B = 1 entry points now share the batched code and still validate under their own names."""
    rc = lib.uc_aligned_bilinear_add(None, 128, 20, 30, B_, 128, 128, 2, None)
    assert rc == -1 and lib.uc_last_error().startswith(b"uc_aligned_bilinear_add: bad arguments")
    dyn = (P * 3)(C_, C_, C_)
    hw = (ctypes.c_int * 6)(10, 10, 5, 5, 2, 2)
    st = (ctypes.c_int * 3)(8, 16, 32)
    so = (ctypes.c_float * 3)(64.0, 128.0, 256.0)
    rc = lib.uc_dynamic_masks(A_, B_, 10, 10, 4, 2, dyn, 176, hw, st, so, D_, None, 1, C_, D_, None)
    assert rc == -1 and lib.uc_last_error().startswith(b"uc_dynamic_masks: null pointer")
    rc = lib.uc_dynamic_masks(A_, B_, 10, 10, 4, 2, dyn, 100, hw, st, so, D_, E_, 1, C_, D_, None)
    assert rc == -1 and lib.uc_last_error().startswith(b"uc_dynamic_masks: bad sizes")

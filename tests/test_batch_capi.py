"""The batched entry points (uc_msda_fused_bf16_batched, uc_corr_propagate_batched, uc_head_decode_batched, uc_postprocess_batched)
reject a bad image count, bad per-sequence strides and a workspace too small for the batch with UC_EINVAL and a message, before any
CUDA call (so this runs without a GPU)."""
import ctypes

import pytest

P = ctypes.c_void_p
L = ctypes.c_long
A_, B_, C_, D_ = P(0x100000), P(0x200000), P(0x300000), P(0x400000)  # never dereferenced: validation comes first


@pytest.fixture(scope="module")
def lib():
    from unicorn_b200 import _lib
    lib = _lib.lib()
    lib.uc_last_error.restype = ctypes.c_char_p
    lib.uc_postprocess_workspace_bytes.restype = ctypes.c_long
    lib.uc_postprocess_workspace_bytes_batched.restype = ctypes.c_long
    return lib


def err(lib, rc):
    assert rc == -1, rc
    return lib.uc_last_error()


def test_msda_batched_rejects_bad_batch(lib):
    hw = (ctypes.c_int * 4)(8, 8, 8, 8)
    for B in (0, -2):
        msg = err(lib, lib.uc_msda_fused_bf16_batched(A_, B_, 192, C_, hw, 2, 8, 4, B, None))
        assert msg.startswith(b"uc_msda_fused_bf16_batched:") and b"B must be >= 1" in msg
    assert b"L<=4" in err(lib, lib.uc_msda_fused_bf16_batched(A_, B_, 192, C_, hw, 5, 8, 4, 2, None))


def corr(lib, B, bs_ref=L(64 * 128), bs_cur=L(64 * 128), bs_v=L(64), bs_out=L(64), n_obj=1):
    # 64 reference / current positions of 128 channels per sequence, one value row
    return lib.uc_corr_propagate_batched(A_, 128, bs_ref, 64, B_, 128, bs_cur, 64, 128, 0, C_, 64, bs_v, n_obj, D_, 64, bs_out, B, None)


def test_corr_batched_rejects_bad_batch_and_strides(lib):
    msg = err(lib, corr(lib, 0))
    assert msg.startswith(b"uc_corr_propagate_batched:") and b"B must be >= 1" in msg
    for kw in (dict(bs_ref=L(64 * 128 - 8)),  # sequences overlap
               dict(bs_cur=L(64 * 128 + 4)),  # not a multiple of 8 elements (TMA needs 16-byte strides)
               dict(bs_v=L(63)),
               dict(bs_out=L(0)),
               dict(bs_out=L(127), n_obj=2)):
        assert b"bad per-sequence strides" in err(lib, corr(lib, 3, **kw)), kw
    assert b"n_obj" in err(lib, corr(lib, 2, n_obj=9))


def test_head_decode_batched_rejects_bad_batch_and_strides(lib):
    ro = (P * 3)(A_, A_, A_)
    cl = (P * 3)(B_, B_, B_)
    hw = (ctypes.c_int * 6)(8, 8, 4, 4, 2, 2)
    st = (ctypes.c_int * 3)(8, 16, 32)
    good_ro, good_cl = (L * 3)(64 * 8, 16 * 8, 4 * 8), (L * 3)(64 * 8, 16 * 8, 4 * 8)
    msg = err(lib, lib.uc_head_decode_batched(ro, cl, hw, st, 8, 8, good_ro, good_cl, 1, 0, C_, None))
    assert msg.startswith(b"uc_head_decode_batched:") and b"B must be >= 1" in msg
    short = (L * 3)(64 * 8, 16 * 8 - 1, 4 * 8)
    assert b"bad per-image strides of level 1" in err(lib, lib.uc_head_decode_batched(ro, cl, hw, st, 8, 8, short, good_cl, 1, 2, C_, None))
    assert b"bad per-image strides of level 2" in err(lib, lib.uc_head_decode_batched(ro, cl, hw, st, 8, 8, good_ro, (L * 3)(512, 128, 0), 1, 2, C_, None))
    assert b"null per-image strides" in err(lib, lib.uc_head_decode_batched(ro, cl, hw, st, 8, 8, None, good_cl, 1, 2, C_, None))


def test_postprocess_batched_rejects_bad_batch_and_small_workspace(lib):
    A = 2100
    one = lib.uc_postprocess_workspace_bytes(A)
    assert lib.uc_postprocess_workspace_bytes_batched(A, 1) == one
    assert lib.uc_postprocess_workspace_bytes_batched(A, 4) == 4 * one
    assert lib.uc_postprocess_workspace_bytes_batched(A, 0) == 0

    def call(B, nbytes):
        return lib.uc_postprocess_batched(A_, A, 1, ctypes.c_float(0.001), ctypes.c_float(0.65), 3, B, B_, L(nbytes), C_, D_, None, None)

    msg = err(lib, call(0, 4 * one))
    assert msg.startswith(b"uc_postprocess_batched:") and b"B must be >= 1" in msg
    msg = err(lib, call(4, 4 * one - 1))
    assert b"workspace too small" in msg and b"4 images of 2100 anchors" in msg
    assert b"workspace too small" in err(lib, call(2, one))

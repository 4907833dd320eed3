"""The batched MOT entry points (uc_sample_embed_batched, uc_copy_rows_if_batched) reject a bad image count, null pointers, per-image
strides smaller than one image and (for the row copy) unaligned rows with UC_EINVAL and a message prefixed by the entry point's name,
before any CUDA call (so this runs without a GPU)."""
import ctypes

import pytest

P = ctypes.c_void_p
L = ctypes.c_long
A_, B_, C_, D_ = (P(0x100000 * k) for k in range(1, 5))  # never dereferenced: validation comes first


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


def test_library_exports_the_batched_mot_entry_points(lib):
    assert hasattr(lib, "uc_sample_embed_batched") and hasattr(lib, "uc_copy_rows_if_batched")


def se(lib, B, embed=A_, boxes=B_, count=C_, out=D_, bs_embed=40 * 40 * 128, bs_boxes=100 * 7, bs_out=100 * 128, n_max=100, ldb=7):
    # 40 x 40 embedding map of 128 channels, up to 100 boxes of 7 floats per image
    return lib.uc_sample_embed_batched(embed, 128, L(bs_embed), 40, 40, 128, 2, boxes, ldb, L(bs_boxes), count, n_max, ctypes.c_float(8.0),
                                       out, L(bs_out), B, None)


def test_sample_embed_batched_rejects_bad_arguments(lib):
    name = b"uc_sample_embed_batched"
    for B in (0, -2):
        assert b"B must be >= 1" in err(lib, se(lib, B), name)
    for kw in (dict(embed=None), dict(boxes=None), dict(count=None), dict(out=None)):
        assert b"null pointer" in err(lib, se(lib, 2, **kw), name), kw
    for kw in (dict(bs_embed=40 * 40 * 128 - 1), dict(bs_boxes=99 * 7), dict(bs_out=100 * 128 - 1)):
        assert b"bad per-image strides" in err(lib, se(lib, 3, **kw), name), kw
    assert b"bad arguments" in err(lib, se(lib, 2, ldb=3), name)
    assert b"bad arguments" in err(lib, se(lib, 2, n_max=-1), name)


def cr(lib, B, flag=A_, gate=None, src=B_, dst=C_, src_ld=256, src_bs=50 * 256, dst_ld=256, dst_bs=50 * 256, row_bytes=256):
    # 50 rows of 256 bytes per image
    return lib.uc_copy_rows_if_batched(flag, gate, 1, src, L(src_ld), L(src_bs), dst, L(dst_ld), L(dst_bs), L(50), row_bytes, B, None)


def test_copy_rows_if_batched_rejects_bad_arguments(lib):
    name = b"uc_copy_rows_if_batched"
    for B in (0, -1):
        assert b"B must be >= 1" in err(lib, cr(lib, B), name)
    for kw in (dict(flag=None), dict(src=None), dict(dst=None)):
        assert b"null pointer" in err(lib, cr(lib, 2, **kw), name), kw
    for kw in (dict(src_bs=49 * 256), dict(dst_bs=50 * 256 - 16)):
        assert b"bad per-image strides" in err(lib, cr(lib, 2, **kw), name), kw
    for kw in (dict(row_bytes=24), dict(src_ld=264), dict(dst=P(0x300008)), dict(src_bs=50 * 256 + 8), dict(dst_bs=50 * 256 + 4)):
        assert b"16-byte aligned rows only" in err(lib, cr(lib, 2, **kw), name), kw


def test_unbatched_entry_points_keep_their_messages(lib):
    """The B = 1 entry points now share the batched kernels and still validate under their own names."""
    rc = lib.uc_sample_embed(None, 128, 40, 40, 128, 2, B_, 7, C_, 100, ctypes.c_float(8.0), D_, None)
    assert rc == -1 and lib.uc_last_error().startswith(b"uc_sample_embed: bad arguments")
    rc = lib.uc_copy_rows_if(A_, 0, B_, L(256), C_, L(256), L(50), 24, None)
    assert rc == -1 and lib.uc_last_error().startswith(b"uc_copy_rows_if: 16-byte aligned rows only")

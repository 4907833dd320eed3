"""The batched MOTS encode (uc_mots_encode_batched) rejects every bad argument with UC_EINVAL and a message prefixed by its name, and by
the image for a per-image argument, before any CUDA call (so this runs without a GPU)."""
import ctypes

import pytest

P, D, L = ctypes.c_void_p, ctypes.c_double, ctypes.c_long
M, O, E, WS, CH, OFF = (P(0x100000 * k) for k in range(1, 7))  # never dereferenced: validation comes first
NAME = b"uc_mots_encode_batched"
N_MAX, HIN, WIN = 8, 800, 1280


@pytest.fixture(scope="module")
def lib():
    from unicorn_b200 import _lib
    lib = _lib.lib()
    lib.uc_last_error.restype = ctypes.c_char_p
    lib.uc_mots_encode_workspace_bytes.restype = ctypes.c_long
    return lib


def encode(lib, k=(4, 0, 8), H=(1080, 480, 720), W=(1920, 640, 1280), r=None, B=None, masks=M, bs=N_MAX * HIN * WIN, n_max=N_MAX,
           order=O, emit=E, work=WS, wbytes=None, chars=CH, cap=1000, offsets=OFF, tables=True):
    B = len(k) if B is None else B
    r = [min(HIN / h, WIN / w) for h, w in zip(H, W)] if r is None else r
    if wbytes is None:
        wbytes = lib.uc_mots_encode_workspace_bytes(sum(k), max(H), max(W))
    arr = lambda t, v: (t * len(v))(*v) if tables else None  # noqa: E731
    rc = lib.uc_mots_encode_batched(masks, L(bs), n_max, HIN, WIN, B, arr(ctypes.c_int, k), arr(ctypes.c_int, H), arr(ctypes.c_int, W),
                                    arr(D, r), order, emit, ctypes.c_float(0.3), work, L(wbytes), chars, L(cap), offsets, None)
    return rc, lib.uc_last_error()


def rejected(lib, **kw):
    rc, msg = encode(lib, **kw)
    assert rc == -1 and msg.startswith(NAME + b":"), (kw, rc, msg)
    return msg


def test_library_exports_the_batched_encode(lib):
    assert hasattr(lib, "uc_mots_encode_batched") and hasattr(lib, "uc_mots_encode")


def test_null_pointers(lib):
    for kw in (dict(masks=None), dict(order=None), dict(emit=None), dict(offsets=None), dict(work=None), dict(chars=None),
               dict(tables=False)):
        assert rejected(lib, **kw) == NAME + b": null pointer", kw
    # no instance in any image: the workspace may be null; no capacity: the chars may be null (n_max = 0 still fails, later)
    assert b"bad sizes" in rejected(lib, k=(0, 0, 0), work=None, n_max=0)
    assert b"bad sizes" in rejected(lib, cap=0, chars=None, n_max=0)


def test_image_count(lib):
    for B in (0, -1, 65):
        assert b"B = %d must be in 1..64" % B in rejected(lib, k=(0,) * max(B, 1), H=(480,) * max(B, 1), W=(640,) * max(B, 1), B=B)


def test_sizes_and_counts(lib):
    for kw in (dict(n_max=0), dict(bs=N_MAX * HIN * WIN - 1)):
        rejected(lib, **kw)
    assert b"bad per-image stride" in rejected(lib, bs=N_MAX * HIN * WIN - 1)
    for kw in (dict(H=(1080, 0, 720), r=(0.6, 1.0, 1.0)), dict(W=(1920, 640, -3), r=(0.6, 1.0, 1.0)), dict(r=(0.6, 0.0, 1.0)),
               dict(r=(0.6, 1.0, -1.0))):
        msg = rejected(lib, **kw)
        assert b"bad sizes" in msg and (b"image 1" in msg or b"image 2" in msg), (kw, msg)
    assert rejected(lib, k=(4, 9, 0)).startswith(NAME + b": image 1: k = 9 must be in 0..n_max (8)")
    assert rejected(lib, k=(4, 0, -1)).startswith(NAME + b": image 2: k = -1 must be in 0..n_max (8)")
    assert b"negative capacity" in rejected(lib, cap=-1)


def test_alignment_workspace_and_empty_resize(lib):
    for kw in (dict(masks=P(0x100002)), dict(order=P(0x300001)), dict(offsets=P(0x600004)), dict(work=P(0x400008))):
        assert b"aligned" in rejected(lib, **kw), kw
    assert b"workspace too small" in rejected(lib, wbytes=16)
    assert rejected(lib, r=(0.6, 1e4, 1.0)).startswith(NAME + b": image 1: the resized mask is empty")

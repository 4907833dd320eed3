"""Argument validation of uc_vos_aggregate_batched (the VOS result assembly of several videos in one launch): every call here is
rejected with UC_EINVAL and a message prefixed by the entry point's name before anything is launched, so the pointers are fake
addresses that are never dereferenced and the test runs without a GPU."""
import ctypes

import pytest

from unicorn_b200 import _lib

P = ctypes.c_void_p
EINVAL = -1
HIN, WIN = 320, 320
CAP = 64  # UC_VOS_MAX_VIDEOS
NAME = b"uc_vos_aggregate_batched"


@pytest.fixture(scope="module")
def lib():
    return _lib.lib()


def objects(ids, init=False):
    objs = (_lib.UcVosObject * max(len(ids), 1))()
    for k, oid in enumerate(ids):
        objs[k].id = oid
        if init and k % 2:
            objs[k].init_mask = 0x300000 + 0x1000 * k
        else:
            objs[k].mask = 0x100000 + 0x1000 * k
    return objs


def video(ids=(1, 2), H=240, W=400, r=0.8, soft=0x500000, seg=0x600000, init=False):
    v = _lib.UcVosVideo()
    v._objs = objects(list(ids), init)  # kept alive with the descriptor
    v.objs = ctypes.cast(v._objs, ctypes.POINTER(_lib.UcVosObject))
    v.n, v.H, v.W, v.r = len(ids), H, W, r
    v.soft_out, v.seg_out = soft, seg
    return v


def call(lib, videos, B=None, Hin=HIN, Win=WIN):
    arr = (_lib.UcVosVideo * max(len(videos), 1))(*videos)
    rc = lib.uc_vos_aggregate_batched(arr, len(videos) if B is None else B, Hin, Win, None)
    return rc, lib.uc_last_error()


def rejected(res, *words):
    rc, msg = res
    assert rc == EINVAL, (rc, msg)
    assert msg.startswith(NAME + b":"), msg
    for w in words:
        assert w.encode() in msg, (w, msg)


def test_entry_points_exist(lib):
    assert hasattr(lib, "uc_vos_aggregate_batched") and hasattr(lib, "uc_vos_aggregate")


def test_rejects_bad_video_counts(lib):
    good = [video(), video(init=True)]
    rejected(call(lib, good, B=0), "B = 0 must be in 1..%d" % CAP)
    rejected(call(lib, good, B=-1), "must be in 1..%d" % CAP)
    rejected(call(lib, [video() for _ in range(CAP + 1)]), "B = %d must be in 1..%d" % (CAP + 1, CAP))
    rc, msg = lib.uc_vos_aggregate_batched(None, 1, HIN, WIN, None), lib.uc_last_error()
    rejected((rc, msg), "null pointer")


@pytest.mark.parametrize("n", [0, 17])
def test_rejects_a_video_with_no_or_too_many_objects(lib, n):
    bad = video(ids=list(range(1, n + 1)) if n <= 16 else list(range(1, 17)))
    bad.n = n
    if n > 16:  # a full array of 17 objects, so the count is what is wrong
        bad._objs = objects(list(range(1, 18)))
        bad.objs = ctypes.cast(bad._objs, ctypes.POINTER(_lib.UcVosObject))
    rejected(call(lib, [video(), bad]), "video 1", "1..16 objects")


@pytest.mark.parametrize("oid", [0, 256, -1])
def test_rejects_object_ids_outside_1_to_255(lib, oid):
    rejected(call(lib, [video(), video(), video(ids=(3, oid, 5))]), "video 2", "object ids must be 1..255")


@pytest.mark.parametrize("field,value", [("H", 0), ("W", 0), ("H", -4), ("r", 0.0), ("r", -0.5), ("r", float("nan"))])
def test_rejects_bad_sizes_and_ratios(lib, field, value):
    bad = video()
    setattr(bad, field, value)
    rejected(call(lib, [bad, video()]), "video 0", "bad sizes")


def test_rejects_bad_network_sizes(lib):
    rejected(call(lib, [video()], Hin=0), "bad sizes")
    rejected(call(lib, [video()], Win=-1), "bad sizes")


def test_rejects_null_seg_out_and_objects(lib):
    rejected(call(lib, [video(), video(seg=None)]), "video 1", "objects")
    bad = video()
    bad.objs = None
    rejected(call(lib, [bad]), "video 0")


def test_one_video_keeps_the_one_video_messages(lib):
    objs = objects([1, 0])
    rc = lib.uc_vos_aggregate(objs, 2, HIN, WIN, 240, 400, ctypes.c_float(0.8), P(0x500000), P(0x600000), None)
    assert rc == EINVAL and lib.uc_last_error() == b"uc_vos_aggregate: object ids must be 1..255"
    rc = lib.uc_vos_aggregate(objects([1]), 1, HIN, WIN, 240, 400, ctypes.c_float(0.0), P(0x500000), P(0x600000), None)
    assert rc == EINVAL and lib.uc_last_error() == b"uc_vos_aggregate: bad sizes"

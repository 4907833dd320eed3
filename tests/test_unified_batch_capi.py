"""Argument validation of uc_groupnorm_apply_gather (the shared head stem of the multi-video unified tracker): every call here is
rejected with UC_EINVAL and a message prefixed by the entry point's name before anything is launched, so the pointers are fake
addresses that are never dereferenced and the test runs without a GPU."""
import ctypes

import pytest

from unicorn_b200 import _lib

P = ctypes.c_void_p
EINVAL = -1
HW = 16
N_SRC = 2
# 16-byte aligned, never dereferenced; y lies past x's N_SRC * HW * 256 bf16 pixels so the two do not overlap
X, STATS, W, B_, PRIOR, BETA, SRC_OF = (P(0x100000 * (i + 1)) for i in range(7))
Y = P(0x800000)


@pytest.fixture(scope="module")
def lib():
    return _lib.lib()


def gather(lib, x=X, ldx=256, n_src=N_SRC, stats=STATS, w=W, b=B_, y=Y, ldy=256, B=3, n_plain=1, src_of=SRC_OF, hw=HW, C=256, G=16,
           eps=1e-3, act=_lib.ACT_SILU, prior=PRIOR, beta=BETA):
    rc = lib.uc_groupnorm_apply_gather(x, ldx, n_src, stats, w, b, y, ldy, B, n_plain, src_of, ctypes.c_long(hw), C, G,
                                       ctypes.c_float(eps), act, prior, beta, None)
    return rc, lib.uc_last_error()


def rejected(call, *words):
    rc, msg = call
    assert rc == EINVAL, (rc, msg)
    assert msg.startswith(b"uc_groupnorm_apply_gather:"), msg
    for w in words:
        assert w.encode() in msg, (w, msg)


def test_rejects_bad_image_counts(lib):
    for n_src in (0, -1, 65536):
        rejected(gather(lib, n_src=n_src), "n_src must be in [1, 65535]")
    for B in (0, -1, 65536):
        rejected(gather(lib, B=B, n_plain=0), "B must be in [1, 65535]")
    rejected(gather(lib, n_plain=-1), "n_plain must be in [0, B]")
    rejected(gather(lib, n_plain=4), "n_plain must be in [0, B]")
    rejected(gather(lib, hw=0), "HW must be >= 1")


def test_rejects_null_and_misaligned_pointers(lib):
    for k in ("x", "stats", "w", "b", "y", "src_of"):
        rejected(gather(lib, **{k: None}), "null pointer")
    rejected(gather(lib, x=P(0x100008)), "16-byte aligned")
    rejected(gather(lib, y=P(0x800004)), "16-byte aligned")
    rejected(gather(lib, stats=P(0x200004)), "stats must be 8-byte aligned")
    rejected(gather(lib, prior=P(0x500002)), "prior must be 4-byte aligned")
    rejected(gather(lib, src_of=P(0x700002)), "src_of must be 4-byte aligned")


def test_rejects_overlapping_maps(lib):
    rejected(gather(lib, y=X), "overlap")
    rejected(gather(lib, y=P(0x100000 - 2 * HW * 256)), "overlap")  # y's second image is x's first
    rejected(gather(lib, y=P(0x100000 + 2 * HW * 256)), "overlap")  # y starts on x's second image
    rejected(gather(lib, y=P(0x100000 + 2 * ((N_SRC * HW - 1) * 256 + 248))), "overlap")  # y starts on x's last pixel


def test_rejects_bad_groups_and_channels(lib):
    rejected(gather(lib, G=24), "C % G == 0")
    rejected(gather(lib, G=0), "G must be >= 1")
    rejected(gather(lib, C=252), "multiples of 8")
    rejected(gather(lib, ldx=260), "multiples of 8")
    rejected(gather(lib, ldx=128), "ldx, ldy >= C")
    rejected(gather(lib, ldy=128), "ldy >= C")
    rejected(gather(lib, C=4104, G=8, ldx=4104, ldy=4104), "C too large")


@pytest.mark.parametrize("act", [_lib.ACT_GELU, _lib.ACT_SIGMOID, 5, -1])
def test_rejects_activations_it_does_not_implement(lib, act):
    rejected(gather(lib, act=act), "act must be")


def test_rejects_a_prior_without_beta_and_the_reverse(lib):
    rejected(gather(lib, beta=None), "prior and beta go together")
    rejected(gather(lib, prior=None), "prior and beta go together")
    # images with a prior need one; with every image plain there must be none
    rejected(gather(lib, prior=None, beta=None), "exactly when n_plain < B")
    rejected(gather(lib, n_plain=3), "exactly when n_plain < B")

"""The C-ABI library loads without a GPU, exports every symbol include/unicorn_b200.h declares, and the product path
fails loudly (no CPU / PyTorch fallback) when there is no sm_90 device."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    txt = open(os.path.join(ROOT, "include", "unicorn_b200.h")).read()
    return sorted(set(re.findall(r"UC_API\s+[\w\s\*]+?\b(uc_\w+)\s*\(", txt)))


def test_header_declares_the_path():
    syms = declared_symbols()
    for s in ("uc_conv2d", "uc_msda_forward_f32", "uc_corr_propagate", "uc_postprocess", "uc_dwconv7", "uc_layernorm"):
        assert s in syms


def test_library_exports_every_declared_symbol():
    from unicorn_b200 import _lib
    lib = _lib.lib()
    for s in declared_symbols():
        assert hasattr(lib, s), f"{s} declared in include/unicorn_b200.h but not exported"
    assert lib.uc_version() >= 100


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU behaviour")
def test_no_cpu_fallback():
    from unicorn_b200 import _lib
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.weights import make_state_dict
    lib = _lib.lib()
    assert lib.uc_check_device() != 0
    with pytest.raises(_lib.UnicornB200Error):
        UnicornEngine(make_state_dict("unicorn_track_tiny", 0), "unicorn_track_tiny", device="cpu")
    d = _lib.UcConv2d()
    assert lib.uc_conv2d(ctypes.byref(d), None) != 0  # argument validation, no launch


def test_new_entry_points_validate_arguments_before_any_launch():
    """uc_dwconv7 / uc_dwconv7_mma / uc_convnext_mlp reject bad arguments with UC_EINVAL and a message, without touching the device (so this runs on
    the CPU box): null pointers, aliasing maps, unsupported channel counts, misaligned pointers."""
    from unicorn_b200 import _lib
    lib = _lib.lib()
    lib.uc_last_error.restype = ctypes.c_char_p
    P = ctypes.c_void_p
    a, b, c = P(0x10000), P(0x20000), P(0x30000)  # never dereferenced: validation comes first
    assert lib.uc_dwconv7_mma(None, b, c, 1, 8, 8, 32, None, None) != 0
    assert lib.uc_dwconv7_mma(a, b, a, 1, 8, 8, 32, None, None) != 0 and b"in-place" in lib.uc_last_error()
    assert lib.uc_dwconv7_mma(a, b, c, 1, 8, 8, 36, None, None) != 0 and b"multiple of 8" in lib.uc_last_error()
    assert lib.uc_dwconv7_mma(P(0x10008), b, c, 1, 8, 8, 32, None, None) != 0 and b"aligned" in lib.uc_last_error()
    assert lib.uc_dwconv7(a, b, c, c, 1, 8, 8, 36, None, None, None) != 0 and b"multiple of 8" in lib.uc_last_error()
    assert lib.uc_dwconv7(P(0x10008), b, c, c, 1, 8, 8, 32, None, None, None) != 0 and b"aligned" in lib.uc_last_error()
    assert lib.uc_dwconv7(a, b, P(0x30004), c, 1, 8, 8, 32, None, None, None) != 0 and b"aligned" in lib.uc_last_error()
    assert lib.uc_convnext_mlp_supported(192) == 1 and lib.uc_convnext_mlp_supported(768) == 0
    f = ctypes.c_float(1e-6)
    assert lib.uc_convnext_mlp(a, b, c, b, c, c, None, 128, 192, f, None) != 0
    assert lib.uc_convnext_mlp(a, b, c, b, c, c, P(0x40000), 128, 768, f, None) != 0 and b"not supported" in lib.uc_last_error()
    assert lib.uc_convnext_mlp(a, b, c, b, c, c, a, 128, 192, f, None) != 0 and b"different maps" in lib.uc_last_error()
    assert lib.uc_convnext_mlp(a, b, c, b, c, c, P(0x40010), 128, 192, f, None) != 0 and b"aligned" in lib.uc_last_error()
    assert lib.uc_convnext_mlp(a, b, c, b, c, c, P(0x40000), 0, 192, f, None) != 0

"""ctypes binding of libunicorn_b200.so (the C ABI in include/unicorn_b200.h).

The product path has no fallback: if the shared library is missing or a launch fails, this raises.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libunicorn_b200.so")

BF16, F32, F16 = 0, 1, 2
ACT_NONE, ACT_RELU, ACT_GELU, ACT_SILU, ACT_SIGMOID = 0, 1, 2, 3, 4


class UcConv2d(ctypes.Structure):
    _fields_ = [
        ("x", ctypes.c_void_p), ("x_dtype", ctypes.c_int),
        ("B", ctypes.c_int), ("H", ctypes.c_int), ("W", ctypes.c_int), ("Cin", ctypes.c_int), ("ldx", ctypes.c_int),
        ("w", ctypes.c_void_p),
        ("Cout", ctypes.c_int), ("KH", ctypes.c_int), ("KW", ctypes.c_int), ("stride", ctypes.c_int), ("pad", ctypes.c_int),
        ("bias", ctypes.c_void_p), ("act", ctypes.c_int),
        ("gamma", ctypes.c_void_p),
        ("res", ctypes.c_void_p), ("ldres", ctypes.c_int),
        ("y", ctypes.c_void_p), ("ldy", ctypes.c_int), ("y_dtype", ctypes.c_int),
        ("block_n", ctypes.c_int),
        ("gn_stats", ctypes.c_void_p), ("gn_groups", ctypes.c_int),
        ("row_stats", ctypes.c_void_p), ("col_s", ctypes.c_void_p), ("row_eps", ctypes.c_float),
        ("act_after_res", ctypes.c_int),
    ]


class UcVosObject(ctypes.Structure):
    _fields_ = [("mask", ctypes.c_void_p), ("init_mask", ctypes.c_void_p), ("id", ctypes.c_int)]


class UcVosVideo(ctypes.Structure):
    _fields_ = [("objs", ctypes.POINTER(UcVosObject)), ("n", ctypes.c_int), ("H", ctypes.c_int), ("W", ctypes.c_int), ("r", ctypes.c_float),
                ("soft_out", ctypes.c_void_p), ("seg_out", ctypes.c_void_p)]


_lib = None


class UnicornB200Error(RuntimeError):
    pass


def lib():
    """Load the library (once).  Raises if it has not been built: there is no CPU / PyTorch fallback."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise UnicornB200Error(
                f"{LIB_PATH} not found: build it with `python -m unicorn_b200.build` "
                "(unicorn_b200 has no CPU/PyTorch fallback path)")
        _lib = ctypes.CDLL(LIB_PATH)
        _lib.uc_last_error.restype = ctypes.c_char_p
    return _lib


LAUNCHES = 0  # kernels launched through the C ABI (claimed count for bench.py's gpu_launches)


def check(rc, what="", n=1):
    global LAUNCHES
    LAUNCHES += n
    if rc != 0:
        msg = lib().uc_last_error().decode("utf-8", "replace")
        raise UnicornB200Error(f"{what} failed (code {rc}): {msg}")


def stream_ptr():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

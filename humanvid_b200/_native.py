"""ctypes binding of libhv_b200.so (the C ABI in include/hv_b200_ops.h and include/hv_b200.h).

There is no fallback: if the shared library is missing this raises, and every call raises RuntimeError with the
library's message on a non-zero status.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libhv_b200.so")

_lib = None


class Epilogue(C.Structure):
    _fields_ = [
        ("bias", C.c_void_p),
        ("rowvec", C.c_void_p),
        ("rowvec_ld", C.c_int32),
        ("rows_per_group", C.c_int32),
        ("residual", C.c_void_p),
        ("ldr", C.c_int32),
        ("act", C.c_int32),
        ("geglu", C.c_int32),
        ("n_valid", C.c_int32),
    ]


ACT_NONE, ACT_RELU, ACT_SILU, ACT_QUICK_GELU = 0, 1, 2, 3

# enum hv_kind in include/hv_b200.h: hv_config.kind, the network a handle runs
HV_KIND_UNET3D, HV_KIND_POSE_GUIDER, HV_KIND_CAMERA_ENCODER, HV_KIND_UNET2D_REF, HV_KIND_VAE, HV_KIND_CLIP_VISION = 0, 1, 2, 3, 4, 5


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(humanvid_b200 has no non-CUDA fallback)"
            )
        _lib = C.CDLL(LIB_PATH)
        # the entry points Python calls that do not return int
        _lib.hv_ops_last_error.restype = C.c_char_p
        _lib.hv_last_error.restype = C.c_char_p
        _lib.hv_last_error.argtypes = [C.c_void_p]
        _lib.hv_workspace_bytes.restype = C.c_size_t
        _lib.hv_last_launch_count.restype = C.c_int64
    return _lib


def check(status: int, handle=None):
    if status != 0:
        l = lib()
        msg = l.hv_ops_last_error().decode()
        if handle is not None:
            try:
                m2 = l.hv_last_error(handle).decode()
                if m2:
                    msg = m2
            except Exception:
                pass
        raise RuntimeError(f"libhv_b200 error {status}: {msg}")


def ptr(t):
    return C.c_void_p(0) if t is None else C.c_void_p(t.data_ptr())


def stream():
    import torch

    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def i64(v):
    return C.c_int64(int(v))


def i32(v):
    return C.c_int32(int(v))

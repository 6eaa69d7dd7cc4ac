"""ctypes binding of ``libdsu_b200.so`` (C ABI in ``include/dsu_b200.h``).

The library is built in-tree by ``__graft_entry__.build()`` (nvcc, sm_90a).  There is no
fallback: if the shared object is missing or the device is not an sm_90 GPU (H100), calls raise.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libdsu_b200.so")

KIND_GENERATORJ_RIC = 1
KIND_GENERATORJ = 2
PREC_FP16 = 0
PREC_FP16X3 = 1
NORM_NONE, NORM_BATCH, NORM_INSTANCE = 0, 1, 2
E_NOTIMPL = -4

PRECISIONS = {"fp16": PREC_FP16, "fp16x3": PREC_FP16X3}


class DsuConfig(C.Structure):
    _fields_ = [("kind", C.c_int32), ("input_channels", C.c_int32), ("filters", C.c_int32 * 6),
                ("resnet_blocks", C.c_int32), ("use_bias", C.c_int32), ("tanh", C.c_int32),
                ("append_smoothers", C.c_int32), ("norm", C.c_int32), ("precision", C.c_int32),
                ("device", C.c_int32)]


# every symbol declared in include/dsu_b200.h: (restype, argtypes)
_VP, _I32, _SZ = C.c_void_p, C.c_int32, C.c_size_t
SYMBOLS = {
    "dsu_last_error": (C.c_char_p, []),
    "dsu_version": (C.c_char_p, []),
    "dsu_create": (C.c_int, [C.POINTER(DsuConfig), C.POINTER(_VP)]),
    "dsu_destroy": (None, [_VP]),
    "dsu_load_weights": (C.c_int, [_VP, C.c_char_p, _VP, C.POINTER(C.c_int64), _I32, _I32, _I32]),
    "dsu_expected_keys": (C.c_int, [_VP]),
    "dsu_loaded_keys": (C.c_int, [_VP]),
    "dsu_finalize": (C.c_int, [_VP, _VP]),
    "dsu_set_knob": (C.c_int, [_VP, C.c_char_p, _I32]),
    "dsu_set_ric_offsets": (C.c_int, [_VP, _I32, _I32, _VP]),
    "dsu_forward": (C.c_int, [_VP, _VP, _I32, _I32, _I32, _VP, _VP]),
    "dsu_forward_u8": (C.c_int, [_VP, _VP, _VP, _VP, _I32, _I32, _I32, _VP, _VP, _VP]),
    "dsu_forward_u8_host": (C.c_int, [_VP, _VP, _VP, _VP, _I32, _I32, _I32, _VP, _VP]),
    "dsu_workspace_bytes": (_SZ, [_VP, _I32, _I32, _I32]),
    "dsu_forward_launches": (C.c_int, [_VP, _I32, _I32, _I32]),
    "dsu_forward_flops": (C.c_double, [_VP, _I32, _I32, _I32]),
    "dsu_frames_to_tensor": (C.c_int, [_VP, _VP, _VP, _I32, _I32, _I32, _VP, _VP, _VP]),
    "dsu_to_image_space": (C.c_int, [_VP, _VP, _SZ, _VP]),
    "dsu_overlap_edge": (C.c_int, [_VP, _VP, _SZ, _VP]),
    "dsu_compose_rgba": (C.c_int, [_VP, _VP, _I32, _I32, _I32, _VP, _VP]),
    "dsu_pos2edge": (C.c_int, [_VP, _I32, _I32, _I32, _VP, _VP]),
    "dsu_profile_forward": (C.c_int, [_VP, _I32, _I32, _I32, _I32, _VP, C.POINTER(C.c_double), C.POINTER(C.c_double), _I32]),
    "dsu_step_name": (C.c_char_p, [_VP, _I32]),
    "dsu_debug_read": (C.c_int, [_VP, _I32, _I32, _VP, _SZ]),
}

_lib: Optional[C.CDLL] = None


def lib() -> C.CDLL:
    """Load the shared library once; raise loudly when it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "drawingspinup_b200: %s is missing - build it with `python -c 'import __graft_entry__ as g; "
                "g.build()'` (nvcc, sm_90a).  There is no CPU or PyTorch fallback." % LIB_PATH)
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(handle, name)
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def last_error() -> str:
    msg = lib().dsu_last_error()
    return msg.decode("utf-8", "replace") if msg else ""


def check(rc: int, what: str) -> None:
    if rc == 0:
        return
    msg = "%s failed (%d): %s" % (what, rc, last_error())
    if rc == E_NOTIMPL:
        raise NotImplementedError(msg)
    raise RuntimeError(msg)

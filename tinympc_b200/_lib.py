"""Loader for the in-tree CUDA library (tinympc_b200/lib/libtinympc_b200.so).

There is NO CPU fallback: if the library is missing or does not export the ABI the header declares,
importing a solver fails loudly.
"""
from __future__ import annotations

import ctypes as C
import os

from . import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libtinympc_b200.so")
_lib = None


class TinyMPCError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"tinympc_b200 error {code}: {msg}")
        self.code = code


def load():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing - build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `make -C tinympc_b200/csrc`). tinympc_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    missing = [n for n in abi.EXPORTS if not hasattr(lib, n)]
    if missing:
        raise ImportError(f"{LIB_PATH} does not export {missing}")
    vp = C.c_void_p
    lib.tinympc_b200_last_error.restype = C.c_char_p
    lib.tinympc_b200_version.restype = C.c_char_p
    lib.tinympc_b200_default_settings.argtypes = [C.POINTER(abi.Settings)]
    lib.tinympc_b200_precompute_cache.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_double] + [vp] * 11
    lib.tinympc_b200_model_blob_elems.argtypes = [C.c_int32, C.c_int32]
    lib.tinympc_b200_precompute_cache_batch.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int64] + [vp] * 7 + [C.c_int32]
    lib.tinympc_b200_precompute_cache_batch_device.argtypes = [vp, C.c_int64] + [vp] * 9
    lib.tinympc_b200_precompute_sensitivity_batch.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int64] + [vp] * 8 + [C.c_int32]
    lib.tinympc_b200_precompute_sensitivity_batch_device.argtypes = [vp, C.c_int64] + [vp] * 10
    lib.tinympc_b200_create.argtypes = [C.POINTER(abi.Problem), C.c_int32, C.POINTER(vp)]
    lib.tinympc_b200_destroy.argtypes = [vp]
    lib.tinympc_b200_update_settings.argtypes = [vp, C.POINTER(abi.Settings)]
    lib.tinympc_b200_get_settings.argtypes = [vp, C.POINTER(abi.Settings)]
    lib.tinympc_b200_set_mode.argtypes = [vp, C.c_int32, C.c_int32]
    lib.tinympc_b200_solve.argtypes = [vp, C.POINTER(abi.Batch), vp]
    lib.tinympc_b200_solve_host.argtypes = [vp, C.POINTER(abi.Batch)]
    lib.tinympc_b200_rollout.argtypes = [vp, C.POINTER(abi.Batch), C.POINTER(abi.Rollout), vp]
    lib.tinympc_b200_get_stats.argtypes = [vp, C.POINTER(abi.Stats)]
    lib.tinympc_b200_advance.argtypes = [vp, C.c_int64, vp, vp, C.c_int64, vp]
    lib.tinympc_b200_advance_models.argtypes = [vp, C.c_int64, vp, vp, C.c_int64, vp, vp]
    lib.tinympc_b200_advance_plant.argtypes = [vp, C.c_int64, vp, vp, C.c_int64, vp, C.c_int32, vp]
    lib.tinympc_b200_supported.argtypes = [C.c_int32, C.c_int32, C.c_int32]
    for n in abi.EXPORTS:
        if n not in ("tinympc_b200_last_error", "tinympc_b200_version"):
            getattr(lib, n).restype = C.c_int
    lib.tinympc_b200_model_blob_elems.restype = C.c_int64
    _lib = lib
    return lib


def check(rc):
    if rc < 0:
        raise TinyMPCError(rc, load().tinympc_b200_last_error().decode())
    return rc

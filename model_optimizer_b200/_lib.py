"""ctypes binding of the C-ABI in ``include/b200quant.h``.

The product path has NO CPU fallback: if the shared library is missing or a call fails, an
exception is raised.  The library is built in-tree by ``__graft_entry__.build()`` (plain nvcc,
sm_90a only) into ``model_optimizer_b200/lib/libb200quant.so``.
"""

from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_double, c_float, c_int, c_size_t, c_uint64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libb200quant.so")

B200Q_OK = 0
F32, F16, BF16 = 0, 1, 2

_lib = None


class B200QuantError(RuntimeError):
    """A b200quant C-ABI call failed (bad argument, unsupported request or CUDA error)."""


# name -> argtypes; every function returns int status unless listed in _SPECIAL
_P = c_void_p
_SIGNATURES = {
    "b200q_device_info": [_P, _P, _P],
    "b200q_set_tuning": [c_char_p, c_int],
    "b200q_get_tuning": [c_char_p, _P],
    "b200q_set_device": [c_int],
    "b200q_amax_per_tensor": [_P, c_int, c_size_t, _P, _P],
    "b200q_amax_rows": [_P, c_int, c_size_t, c_size_t, c_size_t, _P, _P],
    "b200q_amax_cols": [_P, c_int, c_size_t, c_size_t, _P, _P],
    "b200q_abssum_cols": [_P, c_int, c_size_t, c_size_t, _P, _P],
    "b200q_histogram": [_P, c_int, c_size_t, c_int, _P, c_int, _P, _P],
    "b200q_hist_plan": [_P, c_int, c_int, _P, _P],
    "b200q_amax_per_tensor_multi": [_P, c_int, c_size_t, c_int, _P, _P],
    "b200q_fake_quant_nvfp4_multi": [_P, c_int, c_size_t, c_int, _P, c_int, _P],
    "b200q_collect_fake_quant_nvfp4_multi": [_P, c_int, c_size_t, c_int, _P, _P, c_int, _P],
    "b200q_fake_quant_nvfp4_multi_fixup": [_P, _P, c_int, c_int, _P, _P, c_int, _P, c_int, _P, _P],
    "b200q_hist_search_percentile": [_P, c_int, ctypes.c_double, _P, _P],
    "b200q_hist_search_entropy": [_P, c_int, c_int, c_int, c_int, _P, _P, _P, _P],
    "b200q_hist_search_mse": [_P, _P, c_int, c_int, c_int, c_int, c_int, _P, _P],
    "b200q_histogram_planned": [_P, c_int, c_size_t, c_int, _P, _P, _P],
    "b200q_histogram_ex": [_P, c_int, c_size_t, c_int, _P, c_int, _P, _P, _P, _P],
    "b200q_amax_export": [_P, c_size_t, _P, c_int, _P],
    "b200q_nvfp4_block_log2_hist": [_P, c_int, c_size_t, c_float, c_float, c_int, _P, _P, _P],
    "b200q_nvfp4_block_log2_hist_multi": [_P, c_int, c_size_t, c_int, c_float, c_float, c_int, _P, _P, _P],
    "b200q_fake_quant_int": [_P, _P, c_int, c_size_t, _P, c_int, c_size_t, c_size_t, c_int, c_int, c_int, _P],
    "b200q_fake_quant_fp8": [_P, _P, c_int, c_size_t, _P, c_int, c_size_t, c_size_t, _P],
    "b200q_fake_quant_fp8_eager": [_P, _P, c_int, c_size_t, _P, c_int, c_size_t, c_size_t, _P],
    "b200q_fake_quant_nvfp4": [_P, _P, c_int, c_size_t, c_size_t, _P, c_int, _P],
    "b200q_fake_quant_nvfp4_static": [_P, _P, c_int, c_size_t, c_int, _P, _P, c_int, c_float, _P],
    "b200q_pack_nvfp4": [_P, c_int, c_size_t, c_size_t, c_int, _P, _P, _P, _P, _P],
    "b200q_pack_nvfp4_scale2": [_P, c_int, c_size_t, c_size_t, c_int, _P, _P, _P, _P],
    "b200q_pack_nvfp4_static": [_P, c_int, c_size_t, c_size_t, c_int, _P, _P, c_float, _P, _P, _P, _P],
    "b200q_unpack_nvfp4": [_P, _P, _P, _P, c_int, c_size_t, c_size_t, c_int, _P],
    "b200q_pack_int4_blockwise": [_P, c_int, c_size_t, c_int, _P, _P, _P],
    "b200q_unpack_int4_blockwise": [_P, _P, c_int, c_size_t, c_int, _P, _P],
    "b200q_pack_int4_export": [_P, c_int, c_size_t, c_size_t, _P, c_int, c_int, _P, _P],
    "b200q_pack_fp8": [_P, c_int, c_size_t, _P, c_int, c_size_t, c_size_t, _P, _P],
    "b200q_unpack_fp8": [_P, _P, c_int, c_size_t, c_size_t, _P, c_int, c_size_t, _P],
    "b200q_pack_int8": [_P, c_int, c_size_t, _P, c_int, c_size_t, c_size_t, _P, _P],
    "b200q_unpack_int8": [_P, _P, c_int, c_size_t, c_size_t, _P, c_int, c_size_t, _P],
    "b200q_reduce_keep": [_P, c_int, c_size_t, c_size_t, c_size_t, c_size_t, _P, _P, _P, _P],
    "b200q_pack_nf4": [_P, c_int, c_size_t, c_int, _P, _P, _P, _P],
    "b200q_unpack_nf4": [_P, _P, c_int, c_size_t, c_int, _P, _P],
    "b200q_fake_quant_mx": [_P, _P, c_int, c_size_t, c_size_t, c_int, c_int, _P],
    "b200q_pack_mxfp8": [_P, c_int, c_size_t, c_size_t, _P, _P, _P, _P],
    "b200q_unpack_mxfp8": [_P, _P, c_size_t, c_size_t, _P, c_int, _P],
    "b200q_pack_mxfp4": [_P, c_int, c_size_t, c_int, _P, _P, _P],
    "b200q_unpack_mxfp4": [_P, _P, c_size_t, c_int, _P, c_int, _P],
    "b200q_scale_cols": [_P, _P, c_int, c_size_t, c_size_t, _P, c_int, _P],
    "b200q_awq_scale_fake_quant": [_P, _P, c_int, c_size_t, c_size_t, _P, c_int, c_int, c_int, c_int, _P],
    "b200q_awq_weight_scale_sums": [_P, c_int, c_size_t, c_size_t, c_int, _P, _P],
    "b200q_mse_sweep": [_P, c_int, c_size_t, _P, _P, c_int, c_int, c_int, c_int, _P, _P],
    "b200q_mse_sweep_rows": [_P, c_int, c_size_t, c_size_t, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P, _P],
    "b200q_nvfp4_fp8_scale_sweep": [_P, c_int, c_size_t, _P, _P, _P],
    "b200q_nvfp4_fp8_scale_sweep_ex": [_P, c_int, c_size_t, _P, _P, c_int, _P, _P],
    "b200q_nvfp4_fp8_scale_sweep_hessian": [_P, c_int, c_size_t, c_size_t, _P, _P, c_int, _P, _P, _P],
    "b200q_nvfp4_static_mse_sweep": [_P, c_int, c_size_t, _P, _P, _P, c_int, c_float, _P, _P, _P],
    "b200q_hadamard": [_P, _P, c_int, c_size_t, c_size_t, c_size_t, _P, _P],
    "b200q_fake_quant_nvfp4_rotated": [_P, _P, c_int, c_size_t, c_size_t, c_size_t, c_int, _P, c_int, _P],
    "b200q_gptq_block": [_P, c_size_t, c_size_t, c_int, _P, c_size_t, _P, c_int, _P, c_int, c_size_t, c_size_t,
                         c_size_t, c_int, c_int, c_int, _P, _P],
    "b200q_selftest_fastdiv": [c_uint64, c_size_t, _P],
    "b200q_selftest_e2m1_round": [_P],
}

EXPORTED_SYMBOLS = ("b200q_version", "b200q_last_error", "b200q_convert_to_exmy", *_SIGNATURES.keys())


def load() -> ctypes.CDLL:
    """Load (once) and return the shared library; raises if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise B200QuantError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'`. "
            "There is no CPU fallback."
        )
    lib = ctypes.CDLL(LIB_PATH)
    lib.b200q_version.restype = c_int
    lib.b200q_version.argtypes = []
    lib.b200q_last_error.restype = c_char_p
    lib.b200q_last_error.argtypes = []
    lib.b200q_convert_to_exmy.restype = ctypes.c_float
    lib.b200q_convert_to_exmy.argtypes = [ctypes.c_float, c_int]
    for name, argtypes in _SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the build lost a symbol: fail loudly
        fn.restype = c_int
        fn.argtypes = argtypes
    _lib = lib
    return lib


def call(name: str, *args) -> None:
    """Call ``name`` and raise :class:`B200QuantError` on a non-zero status."""
    lib = load()
    rc = getattr(lib, name)(*args)
    if rc != B200Q_OK:
        msg = lib.b200q_last_error().decode("utf-8", "replace")
        raise B200QuantError(f"{name} failed (status {rc}): {msg}")


def set_tuning(key: str, value: int) -> None:
    call("b200q_set_tuning", key.encode(), int(value))


def get_tuning(key: str) -> int:
    v = c_int(0)
    call("b200q_get_tuning", key.encode(), ctypes.byref(v))
    return v.value


def device_info() -> tuple[int, int, int]:
    sm, ma, mi = c_int(0), c_int(0), c_int(0)
    call("b200q_device_info", ctypes.byref(sm), ctypes.byref(ma), ctypes.byref(mi))
    return sm.value, ma.value, mi.value


__all__ = [
    "B200QuantError",
    "BF16",
    "EXPORTED_SYMBOLS",
    "F16",
    "F32",
    "LIB_PATH",
    "call",
    "device_info",
    "get_tuning",
    "load",
    "set_tuning",
    "c_double",
    "c_float",
]

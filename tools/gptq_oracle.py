"""ctypes loader of tools/gptq_oracle.c (CPU ORACLE -- test infrastructure, not product code).

The shared library is compiled on first use with the host C compiler into ``build/oracle`` of the repository, or into
a temporary directory when the tree is read-only."""

from __future__ import annotations

import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "gptq_oracle.c")
CFLAGS = ["-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-Wall"]
_LIB = None

FMT_INT, FMT_FP8, FMT_NVFP4_STATIC, FMT_NVFP4_DYNAMIC = 0, 1, 2, 3
FMT_FP8_EAGER = 4       # the reference's CPU FP8 rule (fl(1 / amax) * 448); oracle only, pins the CPU fixture
PER_TENSOR_COL_BLOCK = 1 << 62


def build(src: str = _SRC) -> str:
    """Compile ``src`` (a C oracle under tools/, by default this one) once per source digest and return the library
    path."""
    name = os.path.splitext(os.path.basename(src))[0]
    with open(src, "rb") as f:
        digest = hashlib.sha256(f.read() + " ".join(CFLAGS).encode()).hexdigest()[:16]
    for d in (os.path.join(os.path.dirname(_HERE), "build", "oracle"),
              os.path.join(tempfile.gettempdir(), f"b200q-oracle-{os.getuid()}")):
        path = os.path.join(d, f"lib{name}.{digest}.so")
        if os.path.exists(path):
            return path
        try:
            os.makedirs(d, exist_ok=True)
            tmp = f"{path}.{os.getpid()}.tmp"
            subprocess.run(["cc", *CFLAGS, "-o", tmp, src, "-lm"], check=True, capture_output=True)
            os.replace(tmp, path)
            return path
        except (OSError, subprocess.CalledProcessError):
            continue
    raise RuntimeError(f"could not compile tools/{name}.c")


def load():
    global _LIB
    if _LIB is None:
        lib = ctypes.CDLL(build())
        P, S, I = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
        lib.oracle_gptq_block.argtypes = [P, S, S, I, P, S, P, I, P, S, S, S, I, I, I, ctypes.c_float, I]
        lib.oracle_gptq_block.restype = None
        lib.oracle_fake_quant_nvfp4_f32.argtypes = [P, P, S, S, I, P, ctypes.c_float]
        lib.oracle_fake_quant_nvfp4_f32.restype = None
        _LIB = lib
    return _LIB


def gptq_block(w, u, fmt, amax, amax_row_stride=0, amax_col_block=PER_TENSOR_COL_BLOCK, col0=0, num_bits=8,
               unsigned=False, narrow_range=False, global_amax=0.0, fma=False):
    """One GPTQ block on a copy of ``w`` [rows, nb] (fp32) with ``u`` [nb, nb]; returns ``(w_out, e)``.

    ``amax``: fp32 values (any shape, flattened), indexed like ``b200q_gptq_block``.  ``fma``: round the in-block
    update like one fused multiply-add (ATen's CPU ``addr_``) instead of a rounded product then an add (its CUDA
    kernel)."""
    w = np.array(w, dtype=np.float32, order="C", copy=True)
    u = np.ascontiguousarray(u, dtype=np.float32)
    amax = np.ascontiguousarray(np.asarray(amax, dtype=np.float32).reshape(-1))
    rows, nb = w.shape
    assert u.shape[0] >= nb and u.shape[1] >= nb and 1 <= nb <= 128
    e = np.zeros((rows, nb), dtype=np.float32)
    load().oracle_gptq_block(w.ctypes.data, nb, rows, nb, u.ctypes.data, u.shape[1], e.ctypes.data, int(fmt),
                             amax.ctypes.data, int(amax_row_stride), int(amax_col_block), int(col0), int(num_bits),
                             int(bool(unsigned)), int(bool(narrow_range)), ctypes.c_float(float(global_amax)),
                             int(bool(fma)))
    return w, e


def fake_quant_nvfp4(x, fmt, amax, global_amax=0.0):
    """NVFP4 fake quant of a whole fp32 [rows, cols] matrix with the oracle's Q (fmt 2 static: fp32 block amax, one per
    16 elements; fmt 3 dynamic: the per-tensor amax)."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    amax = np.ascontiguousarray(np.asarray(amax, dtype=np.float32).reshape(-1))
    assert x.ndim == 2 and x.shape[1] % 16 == 0
    y = np.empty_like(x)
    load().oracle_fake_quant_nvfp4_f32(x.ctypes.data, y.ctypes.data, x.shape[0], x.shape[1], int(fmt),
                                       amax.ctypes.data, ctypes.c_float(float(global_amax)))
    return y

"""ctypes loader of tools/hessian_sweep_oracle.c (CPU ORACLE -- test infrastructure, not product code).

The Hessian-weighted NVFP4 FP8-scale sweep is a 16 x 16 quadratic form evaluated as a chain of fp32 fused
multiply-adds, which NumPy cannot reproduce, so it is restated in C and built like tools/gptq_oracle.c.  The contract
(the C file's header says the same):

- ``x`` is the fp32 widening of the weight, ``a = |x|``;
- candidate ``k``: ``s = cand_scales[k]``, or 1 when that is 0;
- ``q = e2m1_rne_sat(fl(a / s))`` (IEEE division), ``d = fl(a - fl(q * s))``, ``dw = d`` if ``x >= 0`` else ``-d``;
- ``h_c = fmaf(dw[r], H[j][r][c], h_c)`` for ``r = 0..15``, then ``loss = fmaf(h_c, dw[c], loss)`` for ``c = 0..15``;
- the winner is the first ``k`` with ``loss < best`` (``best`` starts at +inf: NaN losses never win, all-NaN / inf
  gives ``k = 0``), and ``best_amax[row * n_cin + j] = cand_amaxes[k]``.
"""

from __future__ import annotations

import ctypes
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from tools import gptq_oracle

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hessian_sweep_oracle.c")
_LIB = None


def build() -> str:
    return gptq_oracle.build(_SRC)


def load():
    global _LIB
    if _LIB is None:
        lib = ctypes.CDLL(build())
        P, S = ctypes.c_void_p, ctypes.c_size_t
        lib.oracle_hessian_sweep.argtypes = [P, S, S, P, P, P, ctypes.c_int, P, P]
        lib.oracle_hessian_sweep.restype = None
        _LIB = lib
    return _LIB


def hessian_sweep(w, hessian, cand_scales, cand_amaxes, return_losses=False):
    """``best_amax`` [cout * n_cin] of the sweep of ``w`` ([cout, n_cin * 16], the fp32 values of a bf16 / fp16 / fp32
    weight) under ``hessian`` ([n_cin, 16, 16]); with ``return_losses`` also the [n_cand, cout * n_cin] losses."""
    w = np.ascontiguousarray(w, dtype=np.float32)
    h = np.ascontiguousarray(hessian, dtype=np.float32)
    sc = np.ascontiguousarray(np.asarray(cand_scales, dtype=np.float32).reshape(-1))
    am = np.ascontiguousarray(np.asarray(cand_amaxes, dtype=np.float32).reshape(-1))
    assert h.ndim == 3 and h.shape[1:] == (16, 16), h.shape
    n_cin = h.shape[0]
    assert w.ndim == 2 and w.shape[1] == n_cin * 16, (w.shape, h.shape)
    assert sc.size == am.size >= 1
    cout = w.shape[0]
    best = np.empty(cout * n_cin, dtype=np.float32)
    lib = load()
    if return_losses:
        losses = np.empty((sc.size, cout * n_cin), dtype=np.float32)
        lib.oracle_hessian_sweep(w.ctypes.data, cout, n_cin, h.ctypes.data, sc.ctypes.data, am.ctypes.data, sc.size,
                                 best.ctypes.data, losses.ctypes.data)
        return best, losses

    def rows(r):                      # ctypes releases the GIL: row chunks run on all cores
        r1 = min(cout, r + step)
        lib.oracle_hessian_sweep(w[r:r1].ctypes.data, r1 - r, n_cin, h.ctypes.data, sc.ctypes.data, am.ctypes.data,
                                 sc.size, best[r * n_cin:r1 * n_cin].ctypes.data, None)

    workers = os.cpu_count() or 1
    step = max(1, -(-cout // (4 * workers)))
    with ThreadPoolExecutor(workers) as ex:
        list(ex.map(rows, range(0, cout, step)))
    return best


def residual(w, cand_scales):
    """``dw`` [n_cand, n_blocks, 16] as the oracle forms it (every step one fp32 operation, so NumPy is exact here)."""
    x = np.ascontiguousarray(w, dtype=np.float32).reshape(-1, 16)
    a = np.abs(x)
    s = np.asarray(cand_scales, dtype=np.float32).reshape(-1, 1, 1)
    s = np.where(s == 0, np.float32(1), s).astype(np.float32)
    with np.errstate(all="ignore"):
        r = (a[None] / s).astype(np.float32)
        q = np.select([r <= 0.25, r < 0.75, r <= 1.25, r < 1.75, r <= 2.5, r < 3.5, r <= 5.0],
                      [0.0, 0.5, 1.0, 1.5, 2.0, 3.0, 4.0], 6.0).astype(np.float32)
        d = (a[None] - (q * s).astype(np.float32)).astype(np.float32)
    return np.where(x[None] >= 0, d, -d).astype(np.float32)


def loss64(dw, hessian, n_cin):
    """Float64 ``dw^T H dw`` per block and the bound ``sum_bd |dw_b H_bd dw_d|`` (the scale of its fp32 rounding),
    both [n_cand, n_blocks]; ``dw`` from ``residual``."""
    d = dw.astype(np.float64).reshape(dw.shape[0], -1, n_cin, 16)
    h = np.asarray(hessian, dtype=np.float64)
    with np.errstate(all="ignore"):
        loss = np.einsum("krnb,nbd,krnd->krn", d, h, d).reshape(dw.shape[0], -1)
        bound = np.einsum("krnb,nbd,krnd->krn", np.abs(d), np.abs(h), np.abs(d)).reshape(dw.shape[0], -1)
    return loss, bound

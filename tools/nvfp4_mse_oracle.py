"""NumPy oracle of the static NVFP4 per-block multiplier search (CPU ORACLE -- test infrastructure, not product code).

Restates ``b200q_nvfp4_static_mse_sweep`` (include/b200quant.h), i.e. the reference's ``MseCalibrator`` run on the
blocked ``[n_blocks, 16]`` weight of a static NVFP4 quantizer (calib/mse.py:84-172): for every candidate multiplier
``m_k`` the fp32 copy of the weight is fake-quantized with block amax ``fl32(a0 * m_k)`` and an fp32 output
(``oracle_np.fake_quant_nvfp4_static(..., dtype="f32")``), the error is ``F.mse_loss(reduction="none")`` (rounded
difference, rounded square), each block's 16 squares are summed, and ``torch.argmin`` over the candidates (first
NaN, else first minimum) picks ``best_amax = fl32(a0 * m_k*)``.

The block sum has two orders:
- ``"cuda"``: ATen's CUDA ``sum(dim=1)`` over 16 contiguous values (Reduce.cuh: one value per thread of a 16-wide
  block row, then ``block_x_reduce``'s shuffle-down tree with offsets 8, 4, 2, 1) -- what a GPU run of the
  reference computes, and what the kernel computes.
- ``"cpu"``: ATen's CPU ``sum(dim=1)`` (``vectorized_inner_sum`` with 8-lane fp32 vectors: lane ``l`` holds
  ``x[l] + x[l + 8]``, and the 8 lanes are added to 0 one after another) -- what the CPU-generated fixture holds.
  Checked against torch's CPU sum on random rows when the fixture is written.
"""

from __future__ import annotations

import numpy as np

from oracle import oracle_np as o

F32 = np.float32


def block_sum(sq, order="cuda"):
    """Sum of each row of ``sq`` [n, 16] (fp32) in the given ATen order."""
    sq = np.asarray(sq, dtype=F32)
    if order == "cuda":
        t = sq.copy()
        w = 8
        while w:
            t[:, :w] = (t[:, :w] + t[:, w:2 * w]).astype(F32)
            w //= 2
        return t[:, 0].copy()
    if order == "cpu":
        lanes = (sq[:, :8] + sq[:, 8:]).astype(F32)
        acc = np.zeros(sq.shape[0], dtype=F32)
        for e in range(8):
            acc = (acc + lanes[:, e]).astype(F32)
        return acc
    raise ValueError(order)


def block_losses(x, amax0, global_amax, mult, fp8_max_norm=448.0, order="cuda"):
    """loss [n_cand, n_blocks] (fp32) of the search; ``x`` is the weight as fp32 values, 16 per block."""
    xb = np.asarray(x, dtype=F32).reshape(-1, 16)
    a0 = np.asarray(amax0, dtype=F32).reshape(-1)
    out = np.empty((len(mult), xb.shape[0]), dtype=F32)
    with np.errstate(over="ignore", invalid="ignore"):
        for k, m in enumerate(np.asarray(mult, dtype=F32)):
            amax = (a0 * m).astype(F32)
            xq = o.fake_quant_nvfp4_static(xb, amax, F32(global_amax), True, fp8_max_norm, "f32")
            d = (xb - xq).astype(F32)
            out[k] = block_sum((d * d).astype(F32), order)
    return out


def search(x, amax0, global_amax, mult, fp8_max_norm=448.0, order="cuda"):
    """-> (best_amax [n_blocks] fp32, best index [n_blocks], losses [n_cand, n_blocks])."""
    losses = block_losses(x, amax0, global_amax, mult, fp8_max_norm, order)
    best = np.argmin(losses, axis=0)                      # first NaN, else first minimum: torch.argmin's rule
    a0 = np.asarray(amax0, dtype=F32).reshape(-1)
    with np.errstate(over="ignore", invalid="ignore"):
        best_amax = (a0 * np.asarray(mult, dtype=F32)[best]).astype(F32)
    return best_amax, best, losses

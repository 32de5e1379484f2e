"""MseCalibrator on the b200quant engine.

Reference: ``modelopt/torch/quantization/calib/mse.py:31-172``.  Its ``collect`` runs, for each of the
``ceil((stop - start) / step) + 1`` multipliers, a full fake quant of the fp32 copy of the tensor, a squared-error
pass and a reduction (39 x ~4 ATen passes for the defaults).  Here ``collect`` is ONE kernel: every candidate amax
is evaluated in registers from a single read of the tensor (``b200q_mse_sweep`` per tensor, ``b200q_mse_sweep_rows``
per channel / per static block).  ``compute_amax`` keeps the reference's argmin (first minimum) and its
``initial_amax * best_candidate`` product, evaluated by torch with the same operand dtypes.

The reference hands the calibrator an opaque ``quant_func(x, amax)``; a fused kernel needs the format instead.
``MseCalibrator(..., quant_func=partial(_mse_quant_func, quantizer=q))`` (what ``model_calib`` builds,
model_calib.py:640-707) is accepted and the format is read off ``q``; otherwise pass ``num_bits`` /
``unsigned`` / ``narrow_range``.

Static NVFP4 quantizers (E2M1 with E4M3 scales over 16-element blocks, fp32 per-block ``_amax`` and a
``global_amax``; the Four-Over-Six preset among them) are searched per block by ``b200q_nvfp4_static_mse_sweep``:
one launch per weight evaluates every candidate of every block, and returns the reference's argmin (first minimum)
and ``initial_amax * best_candidate`` product per block, so ``compute_amax`` only reshapes it.
"""

from __future__ import annotations

import math

import torch

from .. import ops
from .calibrator import _Calibrator


def is_static_nvfp4_search(quantizer, amax) -> bool:
    """Whether the per-block static NVFP4 search kernel covers ``quantizer`` (the engine's or the reference's):
    static E2M1 blocks of 16 with E4M3 scales, a calibrated ``global_amax``, and an fp32 per-block ``amax`` on CUDA."""
    bs = getattr(quantizer, "_block_sizes", None) or {}
    ints = [k for k in bs if isinstance(k, int)]
    return (bool(getattr(quantizer, "is_nvfp4_static", False)) and ints == [-1] and bs.get(-1) == 16
            and getattr(quantizer, "_global_amax", None) is not None
            and isinstance(amax, torch.Tensor) and amax.dtype == torch.float32 and amax.is_cuda)


class MseCalibrator(_Calibrator):
    """Per-tensor / per-channel MSE amax search (calib/mse.py:31-172)."""

    def __init__(self, amax: torch.Tensor, axis=None, step_size: float = 0.1, start_multiplier: float = 0.25,
                 stop_multiplier: float = 4.0, quant_func=None, error_func=None, *, num_bits=None, unsigned=None,
                 narrow_range=None, round_mult: bool = True):
        super().__init__(num_bits=None, axis=axis, unsigned=None)
        if error_func is not None:
            raise NotImplementedError("b200 MseCalibrator: custom error functions are not supported (squared error only)")
        q = getattr(quant_func, "keywords", {}).get("quantizer") if quant_func is not None else None
        self._nvfp4 = q if q is not None and is_static_nvfp4_search(q, amax) else None
        if q is not None:
            num_bits = q._num_bits if num_bits is None else num_bits
            unsigned = q._unsigned if unsigned is None else unsigned
            narrow_range = q._narrow_range if narrow_range is None else narrow_range
        if num_bits is None:
            raise ValueError("b200 MseCalibrator needs the quantizer (quant_func=partial(..., quantizer=q)) or num_bits")
        if self._nvfp4 is None and not (isinstance(num_bits, int) or tuple(num_bits) == (4, 3)):
            raise NotImplementedError(f"b200 MseCalibrator: num_bits={num_bits} (integer formats and FP8-E4M3 only)")
        self._fmt = (num_bits if isinstance(num_bits, int) else 0, bool(unsigned), bool(narrow_range))
        self._best_amax: torch.Tensor | None = None  # static NVFP4: the per-block result of the one collect
        # torch evaluates `amax[R,1] * candidate(0-dim fp32)` in the amax dtype; on CUDA the candidate is rounded to
        # that dtype first, on CPU it is not (include/b200quant.h, b200q_mse_sweep_rows).  True = what a GPU run of the
        # reference computes; False reproduces the CPU-executed fixtures.
        self._round_mult = bool(round_mult)
        self._initial_amax = amax
        self._num_steps = math.ceil((stop_multiplier - start_multiplier) / step_size) + 1
        self._start_multiplier, self._stop_multiplier = start_multiplier, stop_multiplier
        self._candidates: torch.Tensor | None = None
        self._losses: torch.Tensor | None = None     # [n_cand] fp64 (per tensor) or [n_cand, R] fp32 (per row)
        self._amax = None

    def _generate_candidates(self, device):
        return torch.linspace(self._start_multiplier, self._stop_multiplier, steps=self._num_steps, device=device)

    @torch.no_grad()
    def collect(self, x: torch.Tensor):
        if x.device.type != "cuda":
            raise RuntimeError("b200 MseCalibrator: CUDA tensors only (no CPU fallback)")
        x = x.detach()
        if not x.is_contiguous():
            x = x.contiguous()
        a0 = self._initial_amax
        if self._candidates is None:
            self._candidates = self._generate_candidates(x.device)
        if self._nvfp4 is not None:
            if self._best_amax is not None:
                raise RuntimeError("b200 MseCalibrator: static NVFP4 weights are collected once; call reset() first")
            from ..nn.tensor_quantizer import fp8_max_for_normalization

            q = self._nvfp4
            best = ops.nvfp4_static_mse_sweep(x, a0, q._global_amax, self._candidates, fp8_max_for_normalization(q))
            self._best_amax = best.reshape(a0.shape)
            return
        bits, unsigned, narrow = self._fmt
        r = a0.numel()
        if r == 1:
            # the candidate amax values as torch computes them (0-dim * 0-dim promotes to fp32, [1] * 0-dim stays in
            # the amax dtype): handed to the kernel as multipliers of 1.0
            cand = torch.stack([(a0 * c).reshape(()) for c in self._candidates]).float()
            if self._losses is None:
                self._losses = torch.zeros(self._num_steps, dtype=torch.float64, device=x.device)
            ops.mse_sweep_(self._losses, x, torch.ones(1, device=x.device), cand, bits, unsigned, narrow)
            return
        if x.numel() % r or x.dim() < 1 or x.shape[0] != r or (a0.dim() > 0 and a0.shape[0] != r):
            raise NotImplementedError(f"b200 MseCalibrator: amax {tuple(a0.shape)} for input {tuple(x.shape)} "
                                      "(per-tensor, or one amax per row of the first dim)")
        if self._losses is None:
            self._losses = torch.zeros(self._num_steps, r, dtype=torch.float32, device=x.device)
        ops.mse_sweep_rows_(self._losses, x, a0.reshape(-1), self._candidates, bits, unsigned, narrow,
                            cand_dtype=a0.dtype, round_mult=self._round_mult)

    def reset(self):
        self._best_amax = None
        self._losses = None
        self._candidates = None
        self._amax = None
        self._initial_amax = None

    @torch.no_grad()
    def compute_amax(self, verbose: bool = False):
        if self._best_amax is not None:
            self._amax = self._best_amax
        elif self._losses is None:
            return None
        else:
            self._amax = self._amax_from_losses()
        a0 = self._initial_amax
        if verbose:
            ratio = (self._amax / a0).float()
            print(f"MSE Calibrator: best_amax/initial_amax ratio - mean: {ratio.mean().item():.4f}, "
                  f"min: {ratio.min().item():.4f}, max: {ratio.max().item():.4f}")
        return self._amax

    def _amax_from_losses(self):
        best = torch.argmin(self._losses, dim=0)                      # first minimum, like the reference
        best_candidates = self._candidates[best]
        a0 = self._initial_amax
        if best_candidates.ndim != 0:
            best_candidates = best_candidates.view_as(a0)
        return a0 * best_candidates                                   # calib/mse.py:80-84

    def __repr__(self):
        return f"MseCalibrator({super().__repr__()} steps={self._num_steps})"

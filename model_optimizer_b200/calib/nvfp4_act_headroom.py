"""NVFP4ActHeadroomCalibrator on the b200quant engine.

Reference: ``modelopt/torch/quantization/calib/nvfp4_act_headroom.py:36-205`` -- ``collect`` is a clone +
two reductions (per-block amax) + boolean-mask compaction (a host sync) + log2 + bincount per batch; here it
is ONE kernel (block amax in registers, log2 bin, shared-memory histogram, running max).  ``compute_amax``
is the reference's percentile rule ``max(rho * P_anchor, P_upper)`` on the log2 histogram."""

from __future__ import annotations

import math
import warnings

import torch
import torch.nn.functional as F

from .. import ops
from ..config import FP8_NORMAL_DYNAMIC_RANGE as _FP8_NORMAL_DYNAMIC_RANGE
from .calibrator import _Calibrator
_ANCHOR_FLOOR_RATIO = 1e6


class NVFP4ActHeadroomCalibrator(_Calibrator):
    def __init__(self, num_bits=(2, 1), axis=None, unsigned=False, *, block_size=16, anchor_percentile=1.0,
                 upper_percentile=99.99, rho=16384.0, num_bins=512, log2_min=-40.0, log2_max=40.0):
        super().__init__(num_bits, axis, unsigned)
        if not (0.0 < rho < _FP8_NORMAL_DYNAMIC_RANGE):
            raise ValueError(f"rho must be in (0, {_FP8_NORMAL_DYNAMIC_RANGE}); got {rho}.")
        if not (0.0 < anchor_percentile <= 100.0):
            raise ValueError(f"anchor_percentile must be in (0, 100]; got {anchor_percentile}.")
        if not (0.0 < upper_percentile <= 100.0):
            raise ValueError(f"upper_percentile must be in (0, 100]; got {upper_percentile}.")
        if block_size != 16:
            raise NotImplementedError("block_size must be 16")
        self._anchor_percentile, self._upper_percentile = float(anchor_percentile), float(upper_percentile)
        self._rho, self._num_bins = float(rho), int(num_bins)
        self._log2_min, self._log2_max = float(log2_min), float(log2_max)
        self._hist = None
        self._running_max = None
        self._dtype = None

    @torch.no_grad()
    def collect(self, x: torch.Tensor) -> None:
        if x.device.type != "cuda":
            raise RuntimeError("b200 NVFP4ActHeadroomCalibrator: CUDA tensors only (no CPU fallback)")
        x = x.detach()
        rem = x.shape[-1] % 16
        if rem:
            x = F.pad(x, (0, 16 - rem))
        if self._hist is None:
            self._hist = torch.zeros(self._num_bins, dtype=torch.int64, device=x.device)
            self._running_max = torch.zeros(1, dtype=torch.float32, device=x.device)
            self._dtype = x.dtype
        ops.nvfp4_block_log2_hist_(self._hist, self._running_max, x.contiguous(), self._log2_min, self._log2_max)

    def reset(self):
        self._hist = None
        self._running_max = None

    def _bin_index(self, value: float) -> int:
        # fp32 tensor arithmetic like the reference (:110-114)
        frac = (torch.log2(torch.tensor(value)) - self._log2_min) / (self._log2_max - self._log2_min)
        return int((frac * self._num_bins).floor().long().clamp_(0, self._num_bins - 1).item())

    def _percentile(self, counts, percentile, floor_value=None):
        counts = counts.clone()
        if floor_value is not None and floor_value > 0:
            counts[: self._bin_index(floor_value)] = 0
        total = counts.sum()
        if total <= 0:
            return None
        cdf = torch.cumsum(counts, dim=0)
        idx = int(torch.searchsorted(cdf, percentile / 100.0 * total).clamp(0, self._num_bins - 1).item())
        return float(2.0 ** (self._log2_min + (idx + 0.5) / self._num_bins * (self._log2_max - self._log2_min)))

    def amax_from_host(self, counts: torch.Tensor, rmax: float):
        """``compute_amax`` on host values -- ``counts`` a CPU copy of the histogram, ``rmax`` the running max -- as a
        Python float (exact in fp32), or None.  Lets a caller that holds many histograms copy them in one transfer."""
        if not math.isfinite(rmax):
            raise AssertionError("detected nan/inf values in amax")
        if int(counts.sum()) == 0:
            return None if rmax == 0 else rmax
        counts = counts.float()
        upper = rmax if self._upper_percentile >= 100.0 else self._percentile(counts, self._upper_percentile)
        anchor = self._percentile(counts, self._anchor_percentile, upper / _ANCHOR_FLOOR_RATIO if upper else None) \
            if upper else None
        if not upper or upper <= 0 or not anchor or anchor <= 0:
            return rmax
        headroom = self._rho * anchor
        if headroom <= upper:
            warnings.warn(f"[nvfp4_act_headroom] per-block amax range {upper / anchor:.1f} leaves no headroom at "
                          f"rho={self._rho:g}; the scale falls back to the top of the calibrated range.")
        return max(headroom, upper)

    @torch.no_grad()
    def compute_amax(self):
        if self._hist is None:
            return None
        amax = self.amax_from_host(self._hist.cpu(), float(self._running_max.reshape(())))
        return None if amax is None else torch.tensor(amax, dtype=torch.float32, device=self._hist.device)

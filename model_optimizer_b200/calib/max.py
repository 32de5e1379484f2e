"""MaxCalibrator on the b200quant engine.

Reference: ``modelopt/torch/quantization/calib/max.py:26-94`` -- ``collect`` computes
``reduce_amax(x, axis)`` (two full ATen reductions + abs/maximum) and keeps the running elementwise
max, with three host-synchronising asserts per call.  Here ``collect`` is ONE kernel that folds
|x| max straight into device-resident fp32 slots; the NaN / inf / negative checks of the reference
(max.py:69-77) run once, in ``compute_amax``.
"""

from __future__ import annotations

import torch

from .. import ops
from .calibrator import _Calibrator


def _norm_axis(axis, ndim):
    if axis is None:
        return None
    ax = axis if isinstance(axis, (tuple, list)) else (axis,)
    return tuple(sorted(a % ndim for a in ax))


class MaxCalibrator(_Calibrator):
    """Tracks the running per-tensor / per-channel absolute maximum (fp32 slots on device)."""

    def __init__(self, num_bits=8, axis=None, unsigned=False, track_amax=False):
        super().__init__(num_bits, axis, unsigned)
        self._track_amax = track_amax
        self._amaxs = []
        self._slots: torch.Tensor | None = None
        self._shape = None       # keepdims shape of the result
        self._dtype = None       # dtype of the collected tensors (== dtype of the returned amax)

    @property
    def amaxs(self):
        return self._amaxs

    def collect(self, x: torch.Tensor):
        # (no @torch.no_grad(): the statistics come from a detached tensor and raw kernel launches, and the decorator's
        # context-manager round trip is a quarter of this call's host time)
        if x.device.type != "cuda":
            raise RuntimeError("b200 MaxCalibrator: CUDA tensors only (no CPU fallback)")
        x = x.detach()
        if not x.is_contiguous():
            x = x.contiguous()
        if self._axis is None and self._slots is not None and not self._track_amax:
            ops.amax_per_tensor_(self._slots, x)        # steady state of a per-tensor quantizer: straight to the kernel
            return
        keep = _norm_axis(self._axis, x.dim())
        if keep is None:
            shape = ()
            n_slots, mode, arg = 1, "tensor", None
        elif len(keep) == 1:
            a = keep[0]
            shape = tuple(x.shape[i] if i == a else 1 for i in range(x.dim()))
            n_slots = x.shape[a]
            outer = x.stride(a)
            if outer == 1 and a == x.dim() - 1:
                mode, arg = "cols", None
            else:
                mode, arg = "rows", outer
        elif keep == (0, 2) and x.dim() == 4:
            # 2-D block scales: x is the [A, b1, B, b2] view of a matrix, one amax per (a, b) tile.  The rows of
            # length b2 are reduced by the row kernel; folding the b1 rows of a tile is a max over a tensor
            # b2 times smaller than x
            shape = (x.shape[0], 1, x.shape[2], 1)
            n_slots, mode, arg = x.shape[0] * x.shape[2], "tiles", None
        else:
            raise NotImplementedError(f"MaxCalibrator axis={self._axis}: no B200 kernel for this set of kept axes")
        if self._slots is None:
            self._slots = torch.zeros(n_slots, dtype=torch.float32, device=x.device)
            self._shape, self._dtype = shape, x.dtype
        elif self._slots.numel() != n_slots or self._shape != shape:
            raise RuntimeError("amax shape changed!")  # max.py:82-83
        if mode == "tensor":
            ops.amax_per_tensor_(self._slots, x)
        elif mode == "cols":
            ops.amax_cols_(self._slots, x)
        elif mode == "tiles":
            a, b1, b, b2 = x.shape
            rows = torch.zeros(a * b1 * b, dtype=torch.float32, device=x.device)
            ops.amax_rows_(rows, x, b2)
            torch.maximum(self._slots, rows.view(a, b1, b).amax(dim=1).reshape(-1), out=self._slots)
        else:
            ops.amax_rows_(self._slots, x, arg)
        if self._track_amax:
            self._amaxs.append(self._slots.clone().reshape(shape).cpu().numpy())

    def tensor_slot(self, x: torch.Tensor) -> torch.Tensor:
        """The fp32 slot of a per-tensor calibrator (created for x on first use), for a kernel that folds its own |y|
        max into it in place of ``collect`` (``ops.hadamard``)."""
        if self._axis is not None or self._track_amax:
            raise RuntimeError("tensor_slot: per-tensor calibrators without amax tracking only")
        if self._slots is None:
            self._slots = torch.zeros(1, dtype=torch.float32, device=x.device)
            self._shape, self._dtype = (), x.dtype
        elif self._slots.numel() != 1 or self._shape != ():
            raise RuntimeError("amax shape changed!")
        return self._slots

    def reset(self):
        self._slots = None
        self._shape = None
        self._b200_amax_buf = None       # see nn/shared_input.py: the aliased amax of a shared calibrator is stale now

    @property
    def slots(self):
        """Device fp32 running maxima (what the amax arena all-reduces)."""
        return self._slots

    def compute_amax(self):
        if self._slots is None:
            return None
        bad = ~torch.isfinite(self._slots)
        if bool(bad.any()):  # the one host sync; message as in max.py:69-77
            kind = "nan" if bool(torch.isnan(self._slots).any()) else "inf"
            raise AssertionError(f"detected {kind} values in amax")
        return ops.amax_export(self._slots, self._dtype).reshape(self._shape)

    def __repr__(self):
        return f"MaxCalibrator({super().__repr__()} track_amax={self._track_amax})"

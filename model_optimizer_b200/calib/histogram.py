"""HistogramCalibrator on the b200quant engine.

Reference: ``modelopt/torch/quantization/calib/histogram.py:35-343``.  ``collect`` in the reference
is ``min()`` (sync) -> ``abs()`` -> ``float()`` -> ``max()`` -> ``histc`` (4-5 passes, fp32 copy);
here it is one |x| max kernel, a one-thread planning kernel and one histogram kernel (abs fused, no fp32 copy, no
host synchronisation).  ``compute_amax`` runs the reference's searches as GPU kernels over the histogram.
"""

from __future__ import annotations

import numpy as np
import torch

from .. import ops
from .calibrator import _Calibrator


class HistogramCalibrator(_Calibrator):
    """``collect`` never synchronises with the host: the range-growth decision of the reference (:111-130: first
    batch -> ``[0, x_max]`` in ``num_bins`` bins; a later ``x_max`` above the upper edge -> ``ceil(x_max / width)``
    bins up to the last entry of ``arange(0, x_max + width, width)``) is taken by a one-thread kernel into a
    device-resident plan that the histogram kernel reads.  The histogram buffer has a fixed capacity of
    ``max_growth * num_bins`` bins (the range may grow that much after the first batch); an overflow is recorded on
    the device and reported -- loudly -- by ``compute_amax``, the one place that talks to the host."""

    def __init__(self, num_bits=8, axis=None, unsigned=False, num_bins=2048, grow_method=None,
                 skip_zeros=False, torch_hist=True, max_growth: int = 16):
        super().__init__(num_bits, axis, unsigned)
        if axis is not None:
            raise NotImplementedError("Calibrator histogram collection only supports per tensor scaling")
        if skip_zeros:
            raise NotImplementedError("skip_zeros is not supported by the fused histogram kernel")
        self._num_bins0 = int(num_bins)
        self._capacity = int(num_bins) * int(max_growth)
        self._hist_buf: torch.Tensor | None = None    # fp32 [capacity]
        self._plan: torch.Tensor | None = None        # int32 [8] device plan (see ops.hist_plan_)
        self._xmax: torch.Tensor | None = None        # fp32 [1] scratch: |x| max of the current batch
        self._host = None                              # host copy of the plan, filled by _sync()

    @torch.no_grad()
    def collect(self, x: torch.Tensor):
        if x.device.type != "cuda":
            raise RuntimeError("b200 HistogramCalibrator: CUDA tensors only (no CPU fallback)")
        x = x.detach()
        if self._hist_buf is None:
            self._hist_buf = torch.zeros(self._capacity, dtype=torch.float32, device=x.device)
            self._plan = torch.zeros(8, dtype=torch.int32, device=x.device)
            self._xmax = torch.zeros(1, dtype=torch.float32, device=x.device)
            self._scratch = ops.hist_scratch(x.device)   # 16-bit value-pattern counters
        self._host = None
        self._xmax.zero_()
        ops.amax_per_tensor_(self._xmax, x)                                   # 1: |x| max of the batch
        ops.hist_plan_(self._plan, self._xmax, self._num_bins0, self._capacity)   # 2: range decision, on the device
        ops.histogram_planned_(self._hist_buf, x, self._plan, take_abs=True, scratch=self._scratch)   # 3: binning

    def reset(self):
        self._hist_buf = None
        self._plan = None
        self._host = None

    # ---- host view (one synchronisation) -----------------------------------------------------------------
    def _sync(self):
        if self._host is None and self._plan is not None:
            p = self._plan.cpu()
            f = p.view(torch.float32)
            self._host = {"upper": np.float32(f[0].item()), "width": np.float32(f[1].item()),
                          "xmax_grow": np.float32(f[2].item()), "nbins": int(p[3]), "init": int(p[4]),
                          "overflow": int(p[5]), "n_growths": int(p[6])}
            if self._host["overflow"] == 2:
                raise RuntimeError(
                    "HistogramCalibrator: the first batch was all zeros, so the histogram range [0, 0] has zero width "
                    "and cannot grow to a later batch's |x| max; collect a batch with a non-zero value first")
            if self._host["overflow"]:
                raise RuntimeError(
                    f"HistogramCalibrator: a batch needed more than {self._capacity} bins (the range grew more than "
                    f"{self._capacity // self._num_bins0}x after the first batch); rebuild with a larger max_growth")
        return self._host

    @property
    def _num_bins(self):
        h = self._sync()
        return self._num_bins0 if h is None else h["nbins"]

    @property
    def _calib_hist(self):
        if self._hist_buf is None:
            return None
        return self._hist_buf[: self._sync()["nbins"]]

    @property
    def calib_bin_edges(self):
        """The reference's ``_calib_bin_edges``: ``torch.linspace(0, x_max, n + 1)`` after the first batch,
        ``torch.arange(0, x_max + width, width)`` once the range has grown (:119, :124-126; it may hold one more
        entry than ``nbins + 1``, like the reference's)."""
        h = self._sync()
        if h is None:
            return None
        if h["n_growths"] == 0:
            return torch.linspace(0, float(h["upper"]), self._num_bins0 + 1).numpy()
        # on the histogram's device, like the reference's arange(..., device=x.device): torch's CPU fp32 arange rounds
        # some entries differently
        width = torch.tensor(h["width"])
        return torch.arange(0, (torch.tensor(h["xmax_grow"]) + width).item(), width.item(),
                            device=self._hist_buf.device).cpu().numpy()

    def compute_amax(self, method: str = "percentile", *, stride: int = 1, start_bin: int = 128,
                     percentile: float = 99.99):
        """histogram.py:137-190 -> _compute_amax_entropy / _mse / _percentile (:210-343), each a GPU search over the
        device-resident histogram (one CTA per candidate threshold); only the winning index crosses to the host.

        ``mse``: the reference's call site passes ``(centers, amax, num_bits, unsigned)`` into functions whose third
        positional parameter is ``bias`` (:307-310 vs tensor_quant.py:343-355): as shipped it subtracts ``num_bits``
        and quantizes with ``num_bits=int(unsigned)`` on CPU, shifts by -1 in the CUDA kernel, and raises for
        (4, 3).  This implements the documented intent -- ``fake_tensor_quant(centers, amax, bias=None, num_bits,
        unsigned)`` -- pinned against the reference function with that call repaired (tests/golden)."""
        if self._hist_buf is None:
            return None
        hist = self._calib_hist.contiguous()
        edges = self.calib_bin_edges
        if method == "percentile":
            if percentile < 0 or percentile > 100:
                raise ValueError("Invalid percentile. Must be in range 0 <= percentile <= 100.")
            idx = int(ops.hist_search_percentile(hist, percentile).item())
            return torch.tensor(float(edges[idx]))
        if method == "entropy":
            if not isinstance(self._num_bits, int):
                raise TypeError("entropy calibration needs an integer num_bits")
            nq = 1 << (self._num_bits - 1 + int(self._unsigned))
            div = ops.hist_search_entropy(hist, nq, stride, start_bin)
            n = div.numel()
            last = n - 1 - int(torch.argmin(div.flip(0)).item())             # the LAST minimum (:276)
            return torch.tensor(float(edges[last * stride + start_bin]))
        if method == "mse":
            if isinstance(self._num_bits, int) and self._num_bits >= 0:
                bits = self._num_bits
            elif tuple(self._num_bits) == (4, 3):
                bits = 0
            else:
                raise TypeError("Invalid num_bits. num_bits must be a positive integer or tuple (4,3).")
            e = torch.from_numpy(np.asarray(edges, dtype=np.float32)).to(hist.device)
            centers = ((e[1:] + e[:-1]) / 2).contiguous()
            n = min(centers.numel(), hist.numel())        # a grown range may carry one edge more than bins + 1
            mses = ops.hist_search_mse(hist, centers[:n].contiguous(), bits, self._unsigned, stride, start_bin)
            return centers[start_bin + int(torch.argmin(mses).item()) * stride].clone()
        raise TypeError(f"Unknown calibration method {method}")

"""The histogram oracle against CPU torch: ``o.histc`` (ordinary, zero and overflowing ranges) and the growth edges of
``o.HistogramCalibrator`` (the reference's ``arange(0, x_max + width, width)``, calib/histogram.py:124-126)."""

import numpy as np
import pytest
import torch

from oracle import oracle_np as o

F32 = np.float32


def _away_from_edges(v, lo, hi, bins, margin=1e-3):
    """Values whose bin position (v - lo) * bins / (hi - lo), in fp64, is at least ``margin`` from an integer: there
    any fp32 evaluation order of the formula gives the same bin."""
    pos = (v.astype(np.float64) - float(lo)) * bins / (float(hi) - float(lo))
    frac = pos - np.floor(pos)
    return v[(frac > margin) & (frac < 1 - margin)]


@pytest.mark.parametrize("bins", [7, 512, 2048])
@pytest.mark.parametrize("vmax", [1.0, 0.37, 1e-3, 123.4, 3e30])
def test_histc_matches_torch(bins, vmax):
    rng = np.random.default_rng(bins)
    x = (rng.standard_normal(20000) * F32(vmax) * F32(0.6)).astype(F32)
    x = np.concatenate([_away_from_edges(x, 0, F32(vmax), bins), [F32(-vmax), F32(2 * vmax)]]).astype(F32)
    want = torch.histc(torch.from_numpy(x), bins=bins, min=0, max=float(F32(vmax))).numpy()
    got = o.histc(x, bins, vmax)
    assert got.dtype == np.float32
    assert np.array_equal(got, want)


@pytest.mark.parametrize("bins", [7, 8, 511, 2048])
def test_histc_zero_range(bins):
    """torch.histc with min = max = 0 bins over the data's own min and max, and widens a range that is still empty by 1
    on each side: all zeros (+0 and -0) count in bin ``bins // 2`` of [-1, 1]."""
    zeros = np.concatenate([np.zeros(40, F32), -np.zeros(9, F32)])
    want = torch.histc(torch.from_numpy(zeros), bins=bins, min=0, max=0).numpy()
    got = o.histc(zeros, bins, 0.0)
    assert np.array_equal(got, want)
    assert got[bins // 2] == 49 and got.sum() == 49
    threes = np.full(10, F32(3.0))                        # [2, 4]: bin bins // 2 again
    assert np.array_equal(o.histc(threes, bins, 0.0), torch.histc(torch.from_numpy(threes), bins=bins, min=0, max=0).numpy())
    rng = np.random.default_rng(bins)
    lo, hi = F32(-1.25), F32(2.5)
    x = _away_from_edges(rng.uniform(lo, hi, 5000).astype(F32), lo, hi, bins)
    x = np.concatenate([x, [lo, hi]]).astype(F32)
    want = torch.histc(torch.from_numpy(x), bins=bins, min=0, max=0).numpy()
    assert np.array_equal(o.histc(x, bins, 0.0), want)


@pytest.mark.parametrize("bins", [512, 2048])
def test_histc_overflowing_product_saturates(bins):
    """vmax ~ 1e36: v * bins overflows fp32 for the largest values, which count in the last bin, never in bin 0."""
    vmax = F32(1e36)
    x = np.array([vmax, F32(9e35), F32(np.finfo(F32).max / bins * 1.01), F32(1.0), F32(0.0)], F32)
    with np.errstate(over="ignore"):
        assert np.isinf(x[:3] * F32(bins)).all()
    h = o.histc(x, bins, vmax)
    assert h[-1] == 3 and h[0] == 2 and h.sum() == 5


def test_calibrator_zero_first_batch_then_nonzero_raises():
    """The oracle follows the reference: after an all-zero first batch the bin width is 0 and growth fails."""
    c = o.HistogramCalibrator(64)
    c.collect(np.zeros((4, 16), F32))
    assert c.hist[32] == 64 and c.hist.sum() == 64
    with np.errstate(divide="ignore"), pytest.raises(OverflowError):
        c.collect(np.ones((4, 16), F32))


@pytest.mark.parametrize("seed", range(6))
def test_calibrator_growth_edges_match_torch_arange(seed):
    """o.HistogramCalibrator's grown edges == the reference's ``arange(0, x_max + width, width)``, entry for entry and
    in length (which may be nbins + 2), and its bin count == ``ceil(x_max / width)``.  The reference runs that arange
    on the activations' device, whose fp32 kernel rounds the exact product i * width once; torch evaluates it that way
    in fp64 and rounds the result to fp32."""
    rng = np.random.default_rng(seed)
    c = o.HistogramCalibrator(2048)
    first = F32(rng.uniform(0.1, 3.0))
    c.collect(np.array([first, -first / 2, 0.0], F32))
    for k in range(3):
        width = torch.from_numpy(c.edges[1:2]) - torch.from_numpy(c.edges[0:1])
        x_max = F32(float(c.edges[-1]) * rng.uniform(1.05, 2.5))
        c.collect(np.array([x_max, x_max / 2], F32))
        want = torch.arange(0, (torch.tensor(x_max) + width[0]).item(), width[0].item(), dtype=torch.float64).float()
        # the first growth divides by a host scalar, which torch on the GPU applies as x_max * (1 / width)
        q = torch.tensor(x_max) * torch.reciprocal(width[0]) if k == 0 else torch.tensor(x_max) / width[0]
        assert c.num_bins == int(q.ceil().item())
        assert c.edges.size == want.numel() and c.edges.size in (c.num_bins + 1, c.num_bins + 2), (k, c.edges.size)
        assert np.array_equal(c.edges, want.numpy()), (k, np.flatnonzero(c.edges != want.numpy())[:4])

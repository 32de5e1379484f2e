"""HistogramCalibrator at layer scale, bit for bit against a twin of the reference's collect.

The twin restates the ``torch_hist=True`` branch of the reference ``HistogramCalibrator.collect``
(modelopt/torch/quantization/calib/histogram.py:111-130) in plain torch on the GPU:

* ``abs`` when ``min < 0``, then ``.float()`` (:79-82);
* first batch: ``histc(min=0, max=x_max)`` and ``linspace(0, x_max, n + 1)`` (:117-119);
* a later ``x_max`` above the last edge: ``nbins = ceil(x_max / width)`` in fp32 and
  ``arange(0, x_max + width, width)`` on the data's device (:121-126);
* ``histc`` over the current range, ``hist[:old] += old`` (:128-130).

Next to it the twin keeps EXACT int64 counts: histc's bin formula ``trunc(fl(fl(v * nbins) / upper))`` evaluated
in fp32, ``nbins -> nbins - 1``, values outside ``[0, upper]`` skipped, counted with ``bincount``.  A zero range is
widened to ``[-1, 1]`` as ``torch.histc`` widens it, and a product ``v * nbins`` that overflows fp32 saturates to the
last bin (DESIGN.md section 4, "Histogram ranges").  Those counts stay exact past 2^24, where fp32 counts do not.

Every case runs ``collect`` under ``torch.cuda.set_sync_debug_mode("error")``: collect never synchronises.
"""

import numpy as np
import pytest
import torch

from oracle import oracle_np as o

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16, torch.float32]
DT_IDS = ["bf16", "fp16", "fp32"]
TWO24 = 1 << 24
N_PATTERNS = 32768            # scratch layout (include/b200quant.h): 32768 pattern counters, then per-CTA rows
HOT = 1536                    # patterns in the bf16 hot window (csrc/histogram.cu kHot)
HOT_ROWS = 160                # B200Q_HIST_HOT_ROWS
SMALL_SHAPE = (8, 512, 4096)          # 16.8M elements
BIG_SHAPE = (2, 2048, 14336)          # 58.7M elements: a Llama-3-8B MLP activation of 4096 tokens
ZERO_SHAPE = (4, 512, 4096)           # 8.4M zeros: one bin, below 2^24 after two batches
X07 = float(np.float32(0.7))


# ---------------------------------------------------------------------------------------------------------------
# the twin
# ---------------------------------------------------------------------------------------------------------------
def exact_counts(xf, nbins, upper):
    """int64 histc counts of the fp32 CUDA tensor ``xf`` over [0, upper] (upper: fp32 0-dim tensor)."""
    lo, hi = 0.0, float(upper)
    if hi == lo:                                           # torch.histc widens an empty range to [min - 1, max + 1]
        lo, hi = lo - 1.0, hi + 1.0
    v = xf.reshape(-1)
    keep = (v >= lo) & (v <= hi)
    v = v[keep]
    if lo != 0.0:
        v = v - lo
    den = torch.tensor([hi - lo], dtype=torch.float32, device=xf.device)   # a CUDA tensor: a true IEEE division
    q = (v * nbins) / den                                                # fp32: fl(fl(v * nbins) / upper)
    q = torch.clamp(q, max=float(nbins))                                 # an overflowed product -> the last bin
    b = q.to(torch.int64).clamp_(max=nbins - 1)
    return torch.bincount(b, minlength=nbins)


class Twin:
    def __init__(self, num_bins, histc=True):
        self.num_bins = num_bins
        self.histc = histc             # False: exact counts only (torch.histc must not see an overflowing range)
        self.hist = None
        self.exact = None
        self.edges = None
        self.n_growths = 0

    def collect(self, x):
        if x.min() < 0:
            x = x.abs()
        x = x.float()
        x_max = x.max()
        if self.edges is None:
            self.edges = torch.linspace(0, x_max, self.num_bins + 1)
        elif x_max > self.edges[-1]:
            width = self.edges[1] - self.edges[0]
            self.num_bins = int((x_max / width).ceil().item())
            self.edges = torch.arange(0, x_max + width, width, device=x.device)
            self.n_growths += 1
        upper = self.edges[-1]
        e = exact_counts(x, self.num_bins, upper)
        if self.exact is not None:
            e[: self.exact.numel()] += self.exact
        self.exact = e
        if self.histc:
            h = torch.histc(x, bins=self.num_bins, min=0, max=float(upper))
            if self.hist is not None:
                h[: self.hist.numel()] += self.hist
            self.hist = h

    @property
    def upper(self):
        return float(self.edges[-1])


def collect(c, x):
    """``c.collect(x)`` with any host synchronisation turned into an error."""
    torch.cuda.set_sync_debug_mode("error")
    try:
        c.collect(x)
    finally:
        torch.cuda.set_sync_debug_mode("default")


def both(c, tw, x):
    collect(c, x)
    tw.collect(x)


def check(c, tw, what=""):
    """Collect parity with ``==``: histogram (vs histc and vs the exact counts), edges, bin count, growths."""
    h = c._sync()
    assert h["overflow"] == 0, what
    assert h["n_growths"] == tw.n_growths, what
    assert c._num_bins == tw.num_bins, what
    peak = int(tw.exact.max())
    assert peak < TWO24, f"{what}: a bin holds {peak} >= 2^24, counts would not be exact"
    got = c._calib_hist
    assert got.numel() == tw.exact.numel(), what
    bad = torch.nonzero(got.to(torch.int64) != tw.exact).flatten()
    assert bad.numel() == 0, (f"{what}: {bad.numel()} bins differ from the exact counts, first "
                              f"{bad[:4].tolist()}: got {got[bad[:4]].tolist()} want {tw.exact[bad[:4]].tolist()}")
    if tw.histc:
        assert torch.equal(got, tw.hist), what
    want_e = tw.edges.cpu().numpy()
    got_e = c.calib_bin_edges
    assert got_e.shape == want_e.shape, (what, got_e.shape, want_e.shape)
    assert np.array_equal(got_e, want_e), (what, np.flatnonzero(got_e != want_e)[:4])
    # the 16-bit pattern counters are left zeroed for the next batch
    assert int(torch.count_nonzero(c._scratch[:N_PATTERNS])) == 0, what


def gaussian(shape, dtype, seed, scale=1.0, x_max=None, outliers=None):
    """Gaussian activations; ``outliers``: {channel: multiple of sigma}; ``x_max``: one element set to +-x_max (it must
    be the batch's largest magnitude and representable in ``dtype``)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(shape, generator=g, device="cuda", dtype=torch.float32) * scale
    if outliers:
        for ch, k in outliers.items():
            x[..., ch] = k * scale * torch.sign(x[..., ch])
    if x_max is not None:
        x.clamp_(-0.999 * x_max, 0.999 * x_max)
        x.view(-1)[12345 % x.numel()] = -x_max
    x = x.to(dtype)
    if x_max is not None:
        assert float(x.float().abs().max()) == x_max
    return x


def calibrator(num_bins, max_growth=16):
    from model_optimizer_b200.calib import HistogramCalibrator

    return HistogramCalibrator(8, None, False, num_bins=num_bins, max_growth=max_growth)


def bf16_patterns(x):
    return x.contiguous().view(torch.int16).to(torch.int32) & 0x7FFF


def below_window(x, upper):
    """bf16 elements within the range but below the hot window of 1536 patterns under the top pattern of ``upper``."""
    top = int(np.float32(upper).view(np.uint32)) >> 16
    m = bf16_patterns(x)
    return int(((m <= top) & (top - m >= HOT)).sum())


# ---------------------------------------------------------------------------------------------------------------
# searches on a collected histogram
# ---------------------------------------------------------------------------------------------------------------
def check_searches(c, tw, *, mse_configs=None, mse_strides=(1, 3), entropy_stride=1):
    """percentile / mse / entropy on the calibrator's histogram == the oracle's searches on the twin's; the mse losses
    and entropy divergences in full.  Large histograms take larger strides to keep the numpy oracles affordable."""
    from model_optimizer_b200 import ops

    hist = tw.exact.cpu().numpy()
    edges = tw.edges.cpu().numpy()
    nb = hist.size
    assert edges.size in (nb + 1, nb + 2)
    saved = c._num_bits, c._unsigned
    try:
        for pct in (0.0, 50.0, 99.9, 99.99, 100.0):
            assert float(c.compute_amax("percentile", percentile=pct)) == float(o.hist_amax_percentile(hist, edges, pct)), pct

        hist_d = c._calib_hist.contiguous()
        e = torch.from_numpy(edges[: nb + 1].astype(np.float32)).cuda()
        centers_d = ((e[1:] + e[:-1]) / 2).contiguous()
        for bits, unsigned in mse_configs or [(8, False), (4, False), (8, True), ((4, 3), False)]:
            for stride in mse_strides:
                for start in (0, 128):
                    c._num_bits, c._unsigned = bits, unsigned
                    ob = 0 if bits == (4, 3) else bits
                    losses, centers = o.hist_mse_losses(hist, edges[: nb + 1], ob, unsigned, stride, start)
                    got_l = ops.hist_search_mse(hist_d, centers_d, ob, unsigned, stride, start).cpu().numpy()
                    assert got_l.shape == losses.shape
                    # fp32 losses of fp64 sums taken in another order: at most one fp32 rounding apart
                    assert np.all(np.abs(got_l - losses) <= np.spacing(np.abs(losses))), (bits, unsigned, stride, start)
                    got = float(c.compute_amax("mse", stride=stride, start_bin=start))
                    i_want = int(np.argmin(losses))
                    want = float(centers[start + i_want * stride])
                    if got != want:
                        i_got = int(np.argmin(got_l))
                        assert float(centers[start + i_got * stride]) == got
                        # only a tie within fp64 reordering may move the winner
                        assert abs(float(losses[i_got]) - float(losses[i_want])) <= np.spacing(np.float32(losses[i_want])), \
                            (bits, unsigned, stride, start, got, want, losses[i_got], losses[i_want])

        for bits, unsigned in ((8, False), (4, False), (8, True)):
            c._num_bits, c._unsigned = bits, unsigned
            start = 128
            assert float(c.compute_amax("entropy", stride=entropy_stride, start_bin=start)) == \
                float(o.hist_amax_entropy(hist, edges, bits, unsigned, entropy_stride, start)), (bits, unsigned)
            nq = 1 << (bits - 1 + int(unsigned))
            div = ops.hist_search_entropy(hist_d, nq, entropy_stride, start).cpu().numpy()
            ref = o.hist_entropy_divergences(hist, bits, unsigned, entropy_stride, start)
            fin = np.isfinite(ref)
            assert np.array_equal(np.isfinite(div), fin)
            assert np.allclose(div[fin], ref[fin], rtol=1e-10, atol=1e-14)
    finally:
        c._num_bits, c._unsigned = saved


# ---------------------------------------------------------------------------------------------------------------
# layer-width batches
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("num_bins", [2048, 512])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_layer_width_batches(dtype, num_bins):
    """Six full-width batches: an ungrown start, a batch whose |x| max equals the upper edge exactly (no growth: the
    test is ``>``), two growths, and batches inside the grown range."""
    c, tw = calibrator(num_bins), Twin(num_bins)
    x0 = gaussian(BIG_SHAPE, dtype, 1, x_max=5.5)
    both(c, tw, x0)
    if dtype == torch.bfloat16:
        # the hot kernel ran its full grid: one stored row per CTA
        rows = c._scratch[N_PATTERNS:].view(HOT_ROWS, HOT)
        assert int((rows != 0).any(dim=1).sum()) >= 132
    check(c, tw, "first batch")
    up0 = tw.upper
    assert up0 == 5.5
    both(c, tw, gaussian(SMALL_SHAPE, dtype, 2, x_max=up0))        # x_max == upper: no growth
    check(c, tw, "x_max == upper")
    assert tw.n_growths == 0
    both(c, tw, gaussian(BIG_SHAPE, dtype, 3, scale=1.3))
    check(c, tw, "first growth")
    assert tw.n_growths == 1
    both(c, tw, gaussian(SMALL_SHAPE, dtype, 4, scale=0.7))
    both(c, tw, gaussian(BIG_SHAPE, dtype, 5, scale=1.7))
    check(c, tw, "second growth")
    assert tw.n_growths == 2
    both(c, tw, gaussian(BIG_SHAPE, dtype, 6, scale=1.0))
    check(c, tw, "six batches")
    check_searches(c, tw)


# ---------------------------------------------------------------------------------------------------------------
# LLM-like outliers
# ---------------------------------------------------------------------------------------------------------------
OUTLIER_SHAPE = (4, 512, 4096)       # 8.4M elements: bin 0 stays below 2^24 over three batches
OUTLIERS_300 = {7: 300.0, 1001: -37.5, 4000: 20.0}
OUTLIERS_3000 = {7: 3000.0, 1001: 150.0, 3333: -60.0}


@pytest.mark.parametrize("num_bins", [2048, 512])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_outlier_channels(dtype, num_bins):
    """Gaussian activations with outlier channels at 20-3000 sigma: much of the data falls below the hot window of the
    bf16 path (1536 patterns, values down to upper / 4096).  First at ``nbins <= 4000`` (below-window elements are
    bin 0 and credited to pattern 0), then after a tenfold growth past 4000 bins, where more than half of the elements
    are below the window and go to the global pattern counters with their exact pattern."""
    c, tw = calibrator(num_bins), Twin(num_bins)
    x = gaussian(OUTLIER_SHAPE, dtype, 11, outliers=OUTLIERS_300)
    both(c, tw, x)
    assert c._num_bins <= 4000
    if dtype == torch.bfloat16:
        assert below_window(x, tw.upper) > 0.05 * x.numel()
    check(c, tw, "outliers, nbins <= 4000")
    x = gaussian(OUTLIER_SHAPE, dtype, 12, outliers=OUTLIERS_3000)
    both(c, tw, x)
    assert c._num_bins > 4000
    if dtype == torch.bfloat16:
        assert below_window(x, tw.upper) > 0.5 * x.numel()
    check(c, tw, "outliers, nbins > 4000")
    x = gaussian(OUTLIER_SHAPE, dtype, 13, outliers=OUTLIERS_300)
    both(c, tw, x)
    check(c, tw, "outliers inside the grown range")
    check_searches(c, tw, mse_configs=[(8, False), ((4, 3), False)], mse_strides=(16, 48), entropy_stride=16)


# ---------------------------------------------------------------------------------------------------------------
# growth past 8192 bins, to capacity and beyond
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("num_bins", [2048, 512])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_growth_to_capacity(dtype, num_bins):
    """x_max = 1 gives a bin width of exactly 1 / num_bins.  Growth past kHsBins = 8192 (the fp32 element-wise kernel
    moves bins to global atomics), then to exactly ``capacity = 32 * num_bins`` bins, which fits, then a batch that
    needs ``capacity + 1``: ``compute_amax`` raises."""
    max_growth = 32
    cap = num_bins * max_growth
    c, tw = calibrator(num_bins, max_growth), Twin(num_bins)
    both(c, tw, gaussian(SMALL_SHAPE, dtype, 21, x_max=1.0, scale=0.3))
    both(c, tw, gaussian(SMALL_SHAPE, dtype, 22, x_max=20.0, scale=4.0))
    assert c._num_bins == 20 * num_bins and c._num_bins > 8192
    check(c, tw, "past 8192 bins")
    both(c, tw, gaussian(SMALL_SHAPE, dtype, 23, x_max=32.0, scale=6.0))
    assert c._num_bins == cap
    check(c, tw, "at capacity")
    check_searches(c, tw, mse_configs=[(8, False)], mse_strides=(64, 193), entropy_stride=32)
    collect(c, gaussian(SMALL_SHAPE, dtype, 24, x_max=32.5, scale=6.0))   # ceil(32.5 * num_bins) > capacity
    with pytest.raises(RuntimeError, match="max_growth"):
        c.compute_amax("percentile")


def test_growth_edges_with_an_extra_entry():
    """A width that is not a power of two: growth ``arange`` edges hold ``nbins + 2`` entries for some |x| max (the
    reference's ``NOTE``); edges and every search agree with the twin."""
    c, tw = calibrator(2048), Twin(2048)
    both(c, tw, gaussian(SMALL_SHAPE, torch.float32, 31, x_max=X07))
    w = tw.edges[1] - tw.edges[0]
    cands = X07 * 2.9 + torch.arange(4096, dtype=torch.float32) * 1e-6
    pick = None
    for v in cands.tolist():
        v = float(np.float32(v))
        nb = int((torch.tensor(v, device="cuda") / w).ceil().item())
        if torch.arange(0, torch.tensor(v) + w, w).numel() == nb + 2:
            pick = v
            break
    assert pick is not None
    both(c, tw, gaussian(SMALL_SHAPE, torch.float32, 32, x_max=pick, scale=0.5))
    assert tw.edges.numel() == tw.num_bins + 2
    check(c, tw, "nbins + 2 edges")
    check_searches(c, tw)


def _first_growth_targets(w, lo, n=8192):
    """fp32 |x| max values above ``lo`` where the reference's first growth on the GPU, ``x_max / width`` with ``width``
    a CPU scalar (its edges come from ``linspace`` on the host), computed by torch as ``x_max * (1 / width)``, rounds
    to a different ceil than the true quotient.  The later growths divide two device tensors."""
    v = (torch.tensor(lo, dtype=torch.float32) + torch.arange(n, dtype=torch.float32) * 1e-6).cuda()
    rcp = torch.ceil(v * torch.reciprocal(w).item())         # what a CPU-scalar divisor does on CUDA
    quot = torch.ceil(v / w.cuda())
    assert torch.equal(torch.ceil(v / w), rcp)               # the reference's own expression takes the reciprocal
    return v[rcp != quot].cpu().tolist()


def test_first_growth_bin_count():
    """The first growth's ``ceil(x_max / width)`` at an |x| max where the reciprocal and the quotient round apart."""
    c, tw = calibrator(2048), Twin(2048)
    both(c, tw, gaussian(SMALL_SHAPE, torch.float32, 35, x_max=X07))
    targets = _first_growth_targets(tw.edges[1] - tw.edges[0], X07 * 2.9)
    assert targets
    both(c, tw, gaussian(SMALL_SHAPE, torch.float32, 36, x_max=targets[0], scale=0.5))
    check(c, tw, "first growth, reciprocal")
    w = tw.edges[1] - tw.edges[0]                            # a device tensor now: the second growth divides
    both(c, tw, gaussian(SMALL_SHAPE, torch.float32, 37, x_max=float(np.float32(3.3)), scale=0.7))
    check(c, tw, "second growth")
    assert tw.n_growths == 2 and w.is_cuda


# ---------------------------------------------------------------------------------------------------------------
# odd layouts, reset, two calibrators
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_odd_layouts_and_reset(dtype):
    c, tw = calibrator(2048), Twin(2048)
    g = torch.Generator(device="cuda").manual_seed(41)
    base = torch.randn(3_000_017, generator=g, device="cuda").to(dtype)
    both(c, tw, base[1:])                                    # one element off the 16-byte alignment
    check(c, tw, "offset view")
    both(c, tw, (base[: 1_000_003] * 1.5).to(dtype))         # n % 16 != 0
    check(c, tw, "ragged length")
    both(c, tw, torch.tensor([0.5, -3.0, 2.0, 0.0, 7.5], device="cuda").to(dtype))   # shorter than one vector
    check(c, tw, "five elements")
    t = (torch.randn(4096, 1000, generator=g, device="cuda") * 2.5).to(dtype).t()
    assert not t.is_contiguous()
    both(c, tw, t)
    check(c, tw, "transposed view")
    c.reset()
    tw = Twin(2048)
    both(c, tw, (base[3:] * 0.25).to(dtype))
    both(c, tw, base[5:1_000_000])
    check(c, tw, "after reset")


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_two_calibrators_on_one_stream(dtype):
    """Two calibrators collect alternately on one stream; each equals its own twin, so neither leaves anything in the
    scratch the other could pick up."""
    a, ta = calibrator(2048), Twin(2048)
    b, tb = calibrator(512), Twin(512)
    for k in range(4):
        both(a, ta, gaussian(SMALL_SHAPE, dtype, 50 + k, scale=1.0 + 0.4 * k))
        both(b, tb, gaussian(SMALL_SHAPE, dtype, 60 + k, scale=3.0 - 0.5 * k, outliers={k: 40.0}))
    check(a, ta, "calibrator a")
    check(b, tb, "calibrator b")


# ---------------------------------------------------------------------------------------------------------------
# above 2^24 counts per bin
# ---------------------------------------------------------------------------------------------------------------
def test_bin_above_2_24():
    """bf16, 500-sigma outliers over two 58.7M-element batches: bin 0 holds about 22.6M elements.  fp32 counts are no
    longer exact there.  The pattern path adds one float per in-window pattern of the bin, plus one for the patterns
    below the window, per batch (the integer partials before that are exact u32 sums).  Each add is rounded once,
    by at most half an ulp of the running count, so the error is at most n_adds * ulp(count) / 2 (DESIGN.md section 4)."""
    c, tw = calibrator(2048), Twin(2048, histc=False)
    n_adds = 0
    for seed in (71, 72):
        x = gaussian(BIG_SHAPE, torch.bfloat16, seed, outliers={7: 500.0, 1001: -120.0})
        both(c, tw, x)
        assert tw.n_growths == 0
        upper = np.float32(tw.upper)
        top = int(upper.view(np.uint32)) >> 16
        m = bf16_patterns(x).reshape(-1)
        # histc bin of every distinct pattern present
        pats = torch.unique(m)
        v = (pats.to(torch.int32) << 16).view(torch.float32)
        q = torch.clamp((v * 2048) / torch.tensor([float(upper)], device="cuda"), max=2048.0).to(torch.int64)
        bin0 = (v <= float(upper)) & (q == 0)
        in_window = (top - pats) < HOT
        n_adds += int((bin0 & in_window).sum()) + int(bool((bin0 & ~in_window).any()))
    exact = tw.exact
    assert int(exact[0]) > TWO24
    got = c._calib_hist.to(torch.float64)
    ex = exact.to(torch.float64)
    small = exact < TWO24
    assert torch.equal(got[small], ex[small])
    big = ~small
    ulp = torch.from_numpy(np.spacing(exact[big].cpu().numpy().astype(np.float32)).astype(np.float64)).cuda()
    err = (got[big] - ex[big]).abs()
    tol = n_adds * ulp / 2
    assert bool((err <= tol).all()), (err.tolist(), tol.tolist(), n_adds)


# ---------------------------------------------------------------------------------------------------------------
# degenerate ranges
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("num_bins", [2048, 512, 511])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_zero_range(dtype, num_bins):
    """An all-zero first batch gives the range [0, 0]; torch.histc widens it to [-1, 1] and counts the zeros in bin
    ``nbins // 2``.  A second all-zero batch adds to that bin.  A non-zero batch after it cannot grow a zero-width
    range; compute_amax says so (the reference fails there on ``int(inf)``)."""
    c, tw = calibrator(num_bins), Twin(num_bins)
    z = torch.zeros(ZERO_SHAPE, device="cuda", dtype=dtype)
    z.view(-1)[::7] = -0.0
    both(c, tw, z)
    want = torch.histc(z.float().abs(), bins=num_bins, min=0, max=0)
    assert int(want[num_bins // 2]) == z.numel()
    check(c, tw, "all-zero batch")
    assert torch.equal(c._calib_hist, want)
    both(c, tw, torch.zeros(1000, device="cuda", dtype=dtype))
    check(c, tw, "second all-zero batch")
    assert int(c._calib_hist[num_bins // 2]) == z.numel() + 1000
    collect(c, gaussian((64, 512), dtype, 81))
    with pytest.raises(RuntimeError, match="zero") as e:
        c.compute_amax("percentile")
    assert "max_growth" not in str(e.value)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_zero_range_raw_histogram(dtype):
    """``ops.histogram_`` with range_max = 0: zeros go to bin ``nbins // 2``; non-zero values are outside [0, 0] and
    skipped (documented in ops.histogram_), with and without the pattern scratch."""
    from model_optimizer_b200 import ops

    x = torch.tensor([0.0, -0.0, 0.5, 1.0, 0.0, 3.0] * 1001, device="cuda").to(dtype)
    rng = torch.zeros(1, device="cuda")
    for scratch in (None, ops.hist_scratch(x.device)):
        for nbins in (2048, 9000, 7):
            h = torch.zeros(nbins, device="cuda")
            ops.histogram_(h, x, rng, take_abs=True, scratch=scratch)
            want = torch.zeros(nbins, device="cuda")
            want[nbins // 2] = 3 * 1001
            assert torch.equal(h, want), (nbins, scratch is None, torch.nonzero(h).flatten()[:4].tolist())


@pytest.mark.parametrize("num_bins", [2048, 512])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_range_near_flt_max(dtype, num_bins):
    """upper ~ 1e36: ``v * nbins`` overflows fp32 for the largest values.  They belong in the last bin, not in bin 0.
    Checked against the oracle only: torch.histc on the GPU indexes out of bounds for such a range."""
    c = calibrator(num_bins)
    ref = o.HistogramCalibrator(num_bins)
    g = torch.Generator(device="cuda").manual_seed(91)
    for k, s in enumerate((1e36, 6e35)):
        x = ((torch.rand(256, 1024, generator=g, device="cuda") * 2 - 1) * s).to(dtype)
        x.view(-1)[k] = 1e36 if k == 0 else -6e35
        collect(c, x)
        ref.collect(x.float().cpu().numpy())
    got = c._calib_hist.cpu().numpy()
    assert c._num_bins == ref.num_bins == num_bins
    with np.errstate(over="ignore"):
        assert np.float32(ref.edges[-1]) * np.float32(num_bins) == np.inf
    assert ref.hist[-1] > 0
    assert np.array_equal(got, ref.hist), np.flatnonzero(got != ref.hist)[:8]
    assert np.array_equal(c.calib_bin_edges, ref.edges)
    # the twin's exact counts agree with the oracle (both saturate to the last bin)
    tw = Twin(num_bins, histc=False)
    g = torch.Generator(device="cuda").manual_seed(91)
    for k, s in enumerate((1e36, 6e35)):
        x = ((torch.rand(256, 1024, generator=g, device="cuda") * 2 - 1) * s).to(dtype)
        x.view(-1)[k] = 1e36 if k == 0 else -6e35
        tw.collect(x)
    assert np.array_equal(tw.exact.cpu().numpy(), ref.hist.astype(np.int64))

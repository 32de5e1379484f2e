"""The AWQ fixture (tests/golden/ref_awq.npz, tools/gen_awq_golden.py) checked on its own terms, without a GPU.

- The stored losses reproduce the stored winners under the reference's rules: ``awq_clip`` keeps, per block, the
  first ratio whose loss is strictly smaller than every earlier one (model_calib.py:1788-1798), ``awq_lite`` the
  first alpha of minimum loss (``min`` over the loss dict, :1501).
- In the fp32 INT4 ``awq_clip`` cases every stored loss equals a NumPy fp64 restatement of the loss formula -- the
  stored inputs, the strided token subsample, zero padding to whole blocks, the reference's CPU INT4 fake quant of
  the weight at ``amax * ratio``, the squared difference of the per-block partial outputs averaged over tokens --
  within ``LOSS_RTOL`` (see there), and the restatement's winners equal the stored ones wherever a block is not a
  near-tie.
"""

import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import golden  # noqa: E402
from oracle import oracle_np as o  # noqa: E402

CLIP = ("INT4_BLOCKWISE_WEIGHT_ONLY_CFG", "NVFP4_AWQ_CLIP_CFG", "INT8_DEFAULT_CFG", "FP8_DEFAULT_CFG")
LITE = ("INT4_AWQ_CFG", "NVFP4_AWQ_LITE_CFG")
DTYPES = ("f32", "bf16")
LINEARS = ("l0", "l1", "l2")
MAX_TOKENS = 16            # max_tokens_per_batch of the fixture run
NEAR_TIE = 1e-4            # best and runner-up losses within this relative distance: either winner is right
# fp32 losses against the fp64 restatement.  Each loss is the square of a difference of two fp32 block sums of
# 128 products (quantized and unquantized weight); the difference keeps only the quantization error, a few percent
# of each sum, so the sums' rounding (about sqrt(128) * 2^-24 of their magnitude for random-order errors) is
# amplified ~30x in it and ~60x in its square: a few 1e-6 relative.  The fixture's largest is 1.8e-6 (median 1e-7);
# the bound leaves 10x on that.  A wrong formula (no padding, another token stride, an unscaled amax) is off by far
# more: the closest two ratios of any block differ by 1.4e-3 relative.
LOSS_RTOL = 2e-5


@pytest.fixture(scope="module")
def fx():
    return golden.load("ref_awq")


def clip_winners(loss):
    """model_calib.py:1788-1798 over ratios in order: index of the first strictly smaller loss."""
    best = np.full(loss.shape[1:], np.inf)
    idx = np.zeros(loss.shape[1:], dtype=np.int64)
    for i in range(loss.shape[0]):
        better = loss[i] < best
        best = np.where(better, loss[i], best)
        idx = np.where(better, i, idx)
    return idx


def near_ties(loss):
    """Blocks whose best and runner-up losses are within NEAR_TIE of each other (relative to the best)."""
    s = np.sort(loss.reshape(loss.shape[0], -1).astype(np.float64), axis=0)
    return (s[1] - s[0]) <= NEAR_TIE * np.abs(s[0])


def round_mul(a, r, d):
    """``w_amax * ratio`` as torch computes it: the fp32 product, rounded to the amax dtype."""
    return o.round_to((np.float32(a) * np.float32(r)).astype(np.float32), d)


@pytest.mark.parametrize("d", DTYPES)
@pytest.mark.parametrize("preset", CLIP)
def test_clip_losses_reproduce_winners(fx, preset, d):
    key = f"{preset}/{d}"
    ratios = fx[f"{key}/clip.ratios"] if f"{key}/clip.ratios" in fx else None
    searched = [n for n in LINEARS if f"{key}/{n}.clip.loss" in fx]
    if preset in ("INT8_DEFAULT_CFG", "FP8_DEFAULT_CFG"):
        assert not searched and ratios is None        # no block_sizes: max calibration only
        return
    assert searched == list(LINEARS) and list(ratios) == [0.5, 0.55, 0.6, 0.65, 0.7, 0.75, 0.8, 0.85, 0.9, 0.95, 1.0]
    for n in searched:
        loss, w_amax = fx[f"{key}/{n}.clip.loss"], fx[f"{key}/{n}.clip.w_amax"]
        if int(fx[f"{key}/{n}.clip.num_tokens"]) == 0:
            assert n == "l2" and not np.any(loss) and f"{key}/{n}.clip.best" not in fx
            assert np.array_equal(fx[f"{key}/{n}.weight_quantizer.amax"], w_amax)      # the max amax, unclipped
            assert not fx[f"{key}/{n}.weight_quantizer.enabled"]
            continue
        idx = clip_winners(loss).reshape(w_amax.shape)
        want = round_mul(w_amax, ratios[idx], d)
        assert np.array_equal(fx[f"{key}/{n}.clip.best"], want), (key, n)
        assert np.array_equal(fx[f"{key}/{n}.weight_quantizer.amax"], want), (key, n)
        assert np.any(idx < len(ratios) - 1), (key, n)                                 # clipping pays off somewhere


@pytest.mark.parametrize("d", DTYPES)
@pytest.mark.parametrize("preset", LITE)
def test_lite_losses_reproduce_winners(fx, preset, d):
    key = f"{preset}/{d}"
    alphas = fx[f"{key}/lite.alphas"]
    assert np.allclose(alphas, np.arange(11) / 10, atol=1e-6)
    for n in LINEARS:
        loss, best = fx[f"{key}/{n}.lite.loss"], float(fx[f"{key}/{n}.lite.best_alpha"])
        if n == "l2":                                  # never called: no search, neutral pre_quant_scale
            assert not fx[f"{key}/{n}.lite.enabled"] and np.isnan(best) and not np.any(loss)
            assert np.array_equal(fx[f"{key}/{n}.input_quantizer.pqs"], np.ones(136, np.float32))
            continue
        assert fx[f"{key}/{n}.lite.enabled"]
        assert best == alphas[int(np.argmin(loss))], (key, n)
        s = np.sort(loss)
        assert s[1] - s[0] > NEAR_TIE * s[0], (key, n)  # no near-tie among the alphas of this fixture


def _restated_clip_losses(fx, key, n, w_amax, ratios):
    """fp64 restatement of the per-block clip loss for the INT4 block-128 weight of linear ``n``."""
    d = key.split("/")[1]
    m = f"model/{d}"
    xs = fx[f"{m}/calib"].astype(np.float64)
    if n == "l1":                                      # l1 sees relu(l0(x)), l0 unquantized during the search
        xs = np.maximum(xs @ fx[f"{m}/l0.weight"].astype(np.float64).T + fx[f"{m}/l0.bias"], 0.0)
    w = fx[f"{m}/{n}.weight"]
    co, ci = w.shape
    bs = 128
    pad = (-ci) % bs
    nb = (ci + pad) // bs
    wp = np.pad(w, ((0, 0), (0, pad))).reshape(co * nb, bs)
    out = np.zeros((len(ratios), co, nb))
    for x in xs:
        x = x.reshape(-1, ci)
        x = np.pad(x[0:: max(1, x.shape[0] // MAX_TOKENS)], ((0, 0), (0, pad))).reshape(-1, nb, bs)
        org = np.einsum("tbk,cbk->ctb", x, wp.reshape(co, nb, bs).astype(np.float64))
        for i, r in enumerate(ratios):
            amax = round_mul(w_amax, r, d)                               # [co * nb, 1]
            q = o.tensor_quant_cpu(wp, amax, num_bits=4, narrow_range=False, dtype="f32")
            cur = np.einsum("tbk,cbk->ctb", x, q.reshape(co, nb, bs).astype(np.float64))
            out[i] += ((cur - org) ** 2).mean(axis=1)
    return out


@pytest.mark.parametrize("n", ["l0", "l1"])
def test_int4_clip_losses_match_fp64_restatement(fx, n):
    key = "INT4_BLOCKWISE_WEIGHT_ONLY_CFG/f32"
    ratios = fx[f"{key}/clip.ratios"]
    loss, w_amax = fx[f"{key}/{n}.clip.loss"].astype(np.float64), fx[f"{key}/{n}.clip.w_amax"]
    want = _restated_clip_losses(fx, key, n, w_amax, ratios)
    assert want.shape == loss.shape
    rel = np.abs(loss - want) / np.maximum(np.abs(want), 1e-30)
    assert float(rel.max()) <= LOSS_RTOL, (n, float(rel.max()))
    ties = near_ties(want)
    got_idx, want_idx = clip_winners(loss).ravel(), clip_winners(want).ravel()
    assert np.array_equal(got_idx[~ties], want_idx[~ties]), (n, int(np.sum(got_idx[~ties] != want_idx[~ties])))


def test_near_tie_count(fx):
    """The number of near-tie blocks the GPU comparison may resolve either way: few, and reported."""
    counts = {}
    for preset in ("INT4_BLOCKWISE_WEIGHT_ONLY_CFG", "NVFP4_AWQ_CLIP_CFG"):
        for d in DTYPES:
            key = f"{preset}/{d}"
            for n in ("l0", "l1"):
                ties = near_ties(fx[f"{key}/{n}.clip.loss"])
                counts[f"{key}/{n}"] = (int(ties.sum()), ties.size)
    print("awq_clip near-ties (blocks, of):", counts)
    tied = sum(t for t, _ in counts.values())
    total = sum(s for _, s in counts.values())
    assert tied <= 0.03 * total, counts

"""The mirror's ``awq_clip`` and ``awq_lite`` on the GPU against the reference's CPU run (tests/golden/ref_awq.npz,
tools/gen_awq_golden.py): the 3-linear model (an aligned cin, a ragged cin, a linear the forward never calls) under
``awq_clip`` x {INT4 block-128, NVFP4, INT8 per-channel, FP8 per-tensor} and ``awq_lite`` x {INT4, NVFP4}, in fp32
and bf16.  The fixture is the only source of truth here.  Four kinds of check:

- structure, exactly: which quantizers are enabled and hold an ``_amax`` (shape and dtype), which linears were
  searched, which hold a ``_pre_quant_scale`` (the all-ones neutral scale of the never-called linear included);
- maxima, bit for bit: every weight amax that is a plain maximum and every input amax of the data itself (a max does
  not depend on summation order); the input amax of ``l1`` is the max of ``l0``'s output, a GEMM that the GPU sums
  in another order, so it may be a few ulps away;
- the search: each loss within a relative tolerance (the GPU sums in another order than the CPU), and the same
  winners except at blocks the fixture certifies as near-ties;
- values: the smoothed weights within one bf16 ulp, the pre_quant_scales and the held-out output within the
  tolerances of ``test_awq_lite_matches_reference``.

What fails without the host fixes that came with this file: INT8 per-channel weights raised ``TypeError`` (the
clip search ran on weights without blocks) -- every ``INT8_DEFAULT_CFG`` case; FP8 per-tensor weights went through
the clip search (on this data it keeps ratio 1.0, so their amax does not show it) and, like every input quantizer
under awq_clip, their input quantizers got no amax -- ``test_clip_structure`` and ``test_maxima_bit_equal`` of the
FP8 and NVFP4 cases; the never-called linear's weight amax was halved (the first ratio won on all-zero losses) and
its weight quantizer left enabled -- ``test_clip_structure`` / ``test_maxima_bit_equal`` of the INT4 cases; the
never-called linear had no neutral pre_quant_scale -- ``test_lite_structure``; a ragged cin took a per-row instead of
a per-block amax in the AWQ-lite weight scale -- ``test_lite_search`` / ``test_lite_values`` (``l1``).
"""

import numpy as np
import pytest
import torch
from torch import nn

from oracle import golden

pytestmark = pytest.mark.gpu

CLIP = ("INT4_BLOCKWISE_WEIGHT_ONLY_CFG", "NVFP4_AWQ_CLIP_CFG", "INT8_DEFAULT_CFG", "FP8_DEFAULT_CFG")
LITE = ("INT4_AWQ_CFG", "NVFP4_AWQ_LITE_CFG")
DTYPES = ("f32", "bf16")
TD = {"f32": torch.float32, "bf16": torch.bfloat16}
LINEARS = ("l0", "l1", "l2")
QUANTIZERS = ("input_quantizer", "weight_quantizer", "output_quantizer")
CLIP_ARGS = {"max_co_batch_size": 32, "max_tokens_per_batch": 16, "debug": True}
LITE_ARGS = {"alpha_step": 0.1, "debug": True}
NEAR_TIE = 1e-4            # tests/test_awq_cpu.py: best and runner-up within this relative distance
BF16_ULP = 2.0 ** -8       # relative spacing of bf16 (8 significant bits)
# Loss tolerances, GPU against the reference's CPU run.  fp32: both sum the same fp32 values in different orders,
# and the loss squares a difference that keeps only the quantization error of the block sums, which amplifies their
# rounding (tests/test_awq_cpu.py measures 1.8e-6 against fp64): 1e-5.  bf16: the block sums themselves are rounded
# to bf16, so an order change that moves one sum across a rounding boundary moves that token's term by up to one bf16
# ulp of the sum divided by the quantization error (~2^-8 / 3%): the bound is a relative 5e-2 on a single loss.
LOSS_RTOL = {"f32": 1e-5, "bf16": 5e-2}
# held-out output: test_awq_lite_matches_reference's 2e-3 in fp32; in bf16 one bf16 ulp of the output magnitude
# (|y| < 4: 2^-6) on top of it, since a one-ulp difference of a smoothed weight may flip its fake quant
Y_TOL = {"f32": 2e-3, "bf16": 2e-2}
# l1's input amax is the max of l0's output, 128-term fp32 dot products plus a bias.  Summed in another order they
# differ by a few ulps (4.433996 against 4.433997 measured on an H100); 2^-20 allows 8 ulps.  In bf16 the rounded output moves by one ulp at most.
L1_AMAX_RTOL = {"f32": 2.0 ** -20, "bf16": BF16_ULP}


@pytest.fixture(scope="module")
def fx():
    return golden.load("ref_awq")


class Net(nn.Module):
    """tools/gen_awq_golden.py's model: l0 128 -> 136, ReLU, l1 136 -> 64; l2 136 -> 16 is never called."""

    def __init__(self):
        super().__init__()
        self.l0, self.l1, self.l2 = nn.Linear(128, 136), nn.Linear(136, 64), nn.Linear(136, 16)

    def forward(self, x):
        return self.l1(torch.relu(self.l0(x)))


_RUNS = {}


def run(fx, preset, d):
    """The mirror's ``quantize`` with the fixture's algorithm arguments, once per case."""
    if (preset, d) in _RUNS:
        return _RUNS[(preset, d)]
    import model_optimizer_b200.config as cfgs
    from model_optimizer_b200.model_quant import quantize

    model = Net()
    with torch.no_grad():
        for n in LINEARS:
            getattr(model, n).weight.copy_(torch.from_numpy(fx[f"model/{d}/{n}.weight"]))
            getattr(model, n).bias.copy_(torch.from_numpy(fx[f"model/{d}/{n}.bias"]))
    model = model.to(TD[d]).cuda()
    calib = [torch.from_numpy(x).to(TD[d]).cuda() for x in fx[f"model/{d}/calib"]]
    cfg = cfgs.get_preset(preset)
    cfg["algorithm"] = {"method": "awq_clip", **CLIP_ARGS} if preset in CLIP else {"method": "awq_lite", **LITE_ARGS}
    with torch.no_grad():
        quantize(model, cfg, lambda m: [m(x) for x in calib])
        y = model(torch.from_numpy(fx[f"model/{d}/test"]).to(TD[d]).cuda())
    _RUNS[(preset, d)] = (model, host(y))
    return _RUNS[(preset, d)]


def host(t):
    return t.detach().float().cpu().numpy()


def near_ties(loss):
    s = np.sort(loss.reshape(loss.shape[0], -1).astype(np.float64), axis=0)
    return (s[1] - s[0]) <= NEAR_TIE * np.abs(s[0])


def clip_winners(loss):
    best = np.full(loss.shape[1:], np.inf)
    idx = np.zeros(loss.shape[1:], dtype=np.int64)
    for i in range(loss.shape[0]):
        better = loss[i] < best
        best = np.where(better, loss[i], best)
        idx = np.where(better, i, idx)
    return idx


def check_structure(fx, model, key):
    for n in LINEARS:
        lin = getattr(model, n)
        for qn in QUANTIZERS:
            q, p = getattr(lin, qn), f"{key}/{n}.{qn}"
            assert q.is_enabled == bool(fx[p + ".enabled"]), (p, "enabled")
            a = getattr(q, "_amax", None)
            assert (a is not None) == (p + ".amax" in fx), (p, "amax presence")
            if a is not None:
                assert tuple(a.shape) == fx[p + ".amax"].shape, (p, tuple(a.shape), fx[p + ".amax"].shape)
                assert str(a.dtype) == str(fx[p + ".amax_dtype"]), (p, a.dtype, fx[p + ".amax_dtype"])
            s = getattr(q, "_pre_quant_scale", None)
            assert (s is not None) == (p + ".pqs" in fx), (p, "pre_quant_scale presence")
            if s is not None:
                assert tuple(s.shape) == fx[p + ".pqs"].shape and str(s.dtype) == str(fx[p + ".pqs_dtype"]), p


# ---- awq_clip ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", DTYPES)
@pytest.mark.parametrize("preset", CLIP)
def test_clip_structure(fx, preset, d):
    key = f"{preset}/{d}"
    model, _ = run(fx, preset, d)
    check_structure(fx, model, key)
    searched = {n for n in LINEARS if hasattr(getattr(model, n), "awq_clip")}
    assert searched == {n for n in LINEARS if f"{key}/{n}.clip.loss" in fx}
    for n in searched:
        st = getattr(model, n).awq_clip
        assert st.num_tokens == int(fx[f"{key}/{n}.clip.num_tokens"]), n
        assert (getattr(st, "best_clip_val", None) is not None) == (f"{key}/{n}.clip.best" in fx), n


@pytest.mark.parametrize("d", DTYPES)
@pytest.mark.parametrize("preset", CLIP)
def test_maxima_bit_equal(fx, preset, d):
    """Input amaxes, the search's starting weight amax, and every weight amax that no search touched."""
    key = f"{preset}/{d}"
    model, _ = run(fx, preset, d)
    for n in LINEARS:
        lin = getattr(model, n)
        p = f"{key}/{n}.weight_quantizer.amax"
        if f"{key}/{n}.clip.w_amax" in fx:
            assert np.array_equal(host(lin.awq_clip.w_amax), fx[f"{key}/{n}.clip.w_amax"]), n
        if f"{key}/{n}.clip.best" not in fx and p in fx:  # not searched, or searched without tokens: the max
            assert np.array_equal(host(lin.weight_quantizer._amax), fx[p]), (p, "max amax")
        p = f"{key}/{n}.input_quantizer.amax"
        if p in fx:
            assert getattr(lin.input_quantizer, "_amax", None) is not None, (p, "missing")
            got, want = host(lin.input_quantizer._amax), fx[p]
            if n == "l0":                                   # the max of the stored data
                assert np.array_equal(got, want), (p, got, want)
            else:   # the max of l0's output: 128-term dot products that the GPU sums in another order
                assert np.allclose(got, want, rtol=L1_AMAX_RTOL[d], atol=0), (p, got, want)


@pytest.mark.parametrize("d", DTYPES)
@pytest.mark.parametrize("preset", CLIP[:2])
def test_clip_search(fx, preset, d):
    key = f"{preset}/{d}"
    model, y = run(fx, preset, d)
    ratios = list(fx[f"{key}/clip.ratios"])
    ties_total = blocks_total = 0
    for n in ("l0", "l1"):
        st = getattr(model, n).awq_clip
        assert list(st.loss) == ratios
        got = np.stack([host(st.loss[r]) for r in ratios]).astype(np.float64)
        want = fx[f"{key}/{n}.clip.loss"].astype(np.float64)
        assert got.shape == want.shape, n
        rel = np.abs(got - want) / np.maximum(np.abs(want), 1e-30)
        assert float(rel.max()) <= LOSS_RTOL[d], (n, float(rel.max()))
        ties = near_ties(want)
        ties_total, blocks_total = ties_total + int(ties.sum()), blocks_total + ties.size
        gi, wi = clip_winners(got).ravel(), clip_winners(want).ravel()
        assert np.array_equal(gi[~ties], wi[~ties]), (n, int(np.sum(gi[~ties] != wi[~ties])))
        amax, want_amax = host(getattr(model, n).weight_quantizer._amax).ravel(), fx[f"{key}/{n}.weight_quantizer.amax"].ravel()
        keep = np.repeat(~ties, amax.size // ties.size)
        assert np.array_equal(amax[keep], want_amax[keep]), n
    assert ties_total <= 0.03 * blocks_total, (ties_total, blocks_total)
    assert np.allclose(y, fx[f"{key}/y"], atol=Y_TOL[d], rtol=Y_TOL[d]), float(np.abs(y - fx[f"{key}/y"]).max())


@pytest.mark.parametrize("d", DTYPES)
@pytest.mark.parametrize("preset", CLIP[2:])
def test_clip_without_blocks_is_max_calibration(fx, preset, d):
    key = f"{preset}/{d}"
    _, y = run(fx, preset, d)
    assert np.allclose(y, fx[f"{key}/y"], atol=Y_TOL[d], rtol=Y_TOL[d]), float(np.abs(y - fx[f"{key}/y"]).max())


# ---- awq_lite ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", DTYPES)
@pytest.mark.parametrize("preset", LITE)
def test_lite_structure(fx, preset, d):
    key = f"{preset}/{d}"
    model, _ = run(fx, preset, d)
    check_structure(fx, model, key)
    for n in LINEARS:
        st = getattr(model, n).awq_lite                        # every linear with an enabled weight quantizer
        searched = not np.isnan(fx[f"{key}/{n}.lite.best_alpha"])
        assert (st.best_alpha is not None) == searched, n
        if not searched:
            assert np.array_equal(host(getattr(model, n).input_quantizer._pre_quant_scale),
                                  np.ones(getattr(model, n).weight.shape[1], np.float32)), n


@pytest.mark.parametrize("d", DTYPES)
@pytest.mark.parametrize("preset", LITE)
def test_lite_search(fx, preset, d):
    key = f"{preset}/{d}"
    model, _ = run(fx, preset, d)
    alphas = fx[f"{key}/lite.alphas"]
    for n in ("l0", "l1"):
        st = getattr(model, n).awq_lite
        assert np.allclose(st.alphas, alphas, atol=1e-6)
        assert np.allclose(host(st.weight_scale), fx[f"{key}/{n}.lite.weight_scale"], rtol=BF16_ULP if d == "bf16" else 1e-6,
                           atol=0), n
        got, want = host(st.loss).astype(np.float64), fx[f"{key}/{n}.lite.loss"]
        rel = np.abs(got - want) / np.abs(want)
        assert float(rel.max()) <= LOSS_RTOL[d], (n, float(rel.max()))
        assert abs(st.best_alpha - float(fx[f"{key}/{n}.lite.best_alpha"])) < 1e-6, (n, st.best_alpha)


@pytest.mark.parametrize("d", DTYPES)
@pytest.mark.parametrize("preset", LITE)
def test_lite_values(fx, preset, d):
    key = f"{preset}/{d}"
    model, y = run(fx, preset, d)
    for n in LINEARS:
        lin = getattr(model, n)
        w, want = host(lin.weight), fx[f"{key}/{n}.weight_after"]
        assert np.all(np.abs(w - want) <= BF16_ULP * np.abs(want)), (n, float(np.max(np.abs(w - want) / np.abs(want))))
        pqs, want = host(lin.input_quantizer._pre_quant_scale), fx[f"{key}/{n}.input_quantizer.pqs"]
        assert np.allclose(pqs, want, rtol=1e-4 if d == "f32" else BF16_ULP, atol=0), n
        for qn in ("input_quantizer", "weight_quantizer"):
            p = f"{key}/{n}.{qn}.amax"
            if p in fx:
                a = host(getattr(lin, qn)._amax)
                assert np.allclose(a, fx[p], rtol=1e-4 if d == "f32" else BF16_ULP, atol=0), (p, a, fx[p])
    assert np.allclose(y, fx[f"{key}/y"], atol=Y_TOL[d], rtol=Y_TOL[d]), float(np.abs(y - fx[f"{key}/y"]).max())

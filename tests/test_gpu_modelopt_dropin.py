"""The north-star boundary on the GPU: the REAL ``modelopt.torch.quantization.quantize()`` (the unmodified
reference installed into ``baseline/_ref`` by ``__graft_entry__.build()``), once stock -- the reference's own CUDA
extensions (compiled from its sources, ``oracle/build_ref_ext.py``) and its Triton kernels (JIT on the box) -- and
once with this engine plugged in through ``backend.install()`` + ``with_b200_backend`` (backend entry point,
``B200MaxCalibrator`` via the ``calibrator`` field, extension shims, FP8-sweep factory, QTensor packs).

Same tiny HF Llama, same seeded calibration batches.  Bars (written per test):
  * every ``_amax`` / ``_global_amax`` / ``_pre_quant_scale`` buffer bit-equal;
  * fake-quant outputs of every quantizer on a fresh input bit-equal for INT8 / FP8 / INT4, and equal up to exact
    E2M1 rounding ties for NVFP4 (the reference's Triton kernels divide with ``div.full.f32``; its own test skips
    tie vectors, tests/gpu/torch/quantization/test_tensor_quant_cuda.py:243-245);
  * ``mtq.compress`` packed weights and scales bit-exact;
  * ``backend.stats`` proves the b200 arm actually ran the kernels (no silent stock path).

Without the reference installed, the stock arm's results are the golden data ``tests/golden/ref_dropin*.npz`` (the
buffers, logits, digests of the compressed weights, and seeded spread samples of every per-quantizer output and of
the weights)
and the engine arm is this repo's own ``quantize()`` mirror on the same model and batches, held to the same bars.
Those files are what a run with the reference writes when ``DROPIN_GOLDEN_OUT`` names a directory."""

import copy
import functools
import hashlib
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REPORT = {}
GOLDEN = "ref_dropin"
GOLDEN_OUT = os.environ.get("DROPIN_GOLDEN_OUT")   # a run with the reference writes the stock arm's results here
RECORD = {}
SAMPLE = 4096                                      # stored elements per per-quantizer output / weight


class Env(tuple):
    """(mtq, backend) of the reference install, or the stock arm's stored results (``golden``)."""

    def __new__(cls, mtq=None, backend=None, golden=None):
        e = super().__new__(cls, (mtq, backend))
        e.golden = golden
        return e

    @property
    def live(self):
        return self.golden is None


@pytest.fixture(scope="module")
def env():
    from baseline import ref_env

    if not ref_env.available():
        from oracle import golden

        return Env(golden=golden.load(GOLDEN))
    mtq = ref_env.activate()
    loaded = ref_env.use_prebuilt_extensions()
    from model_optimizer_b200 import backend

    REPORT["reference_extensions_prebuilt"] = loaded
    return Env(mtq, backend)


@functools.lru_cache(maxsize=None)
def _spread_index(numel):
    """SAMPLE flat indices spread over a tensor of ``numel`` elements (all of them when it is smaller), seeded by
    the size alone so that both arms and the stored data pick the same ones."""
    if numel <= SAMPLE:
        return torch.arange(numel)
    return torch.randperm(numel, generator=torch.Generator().manual_seed(numel))[:SAMPLE].sort().values


def spread(t):
    """The seeded spread sample of ``t`` (flattened) that the golden data stores."""
    flat = t.reshape(-1)
    return flat[_spread_index(flat.numel()).to(flat.device)]


def _np(t):
    return t.detach().float().cpu().numpy() if t.dtype != torch.float8_e4m3fn else t.view(torch.uint8).cpu().numpy()


def _digest(t):
    return np.frombuffer(hashlib.sha256(t.detach().reshape(-1).contiguous().view(torch.uint8).cpu().numpy().tobytes()).digest(),
                         dtype=np.uint8)


def record(case, kind, name, value):
    """Stock-arm result of a live run, kept for the golden file."""
    if GOLDEN_OUT:
        RECORD[f"{case}/{kind}/{name}"] = value


def stored(env, case, kind):
    """{name: array} of one kind of stored stock-arm result."""
    pre = f"{case}/{kind}/"
    return {k[len(pre):]: env.golden[k] for k in env.golden.files if k.startswith(pre)}


def as_tensor(a, like):
    return torch.from_numpy(np.ascontiguousarray(a)).to(device=like.device).to(like.dtype).reshape(like.shape)


def mirror_quantize(preset, algorithm=None):
    """The engine arm without the reference: this repo's quantize() on the same model and batches."""
    import model_optimizer_b200.config as cfgs
    from model_optimizer_b200.model_quant import quantize

    cfg = copy.deepcopy(getattr(cfgs, preset))
    if algorithm is not None:
        cfg["algorithm"] = algorithm
    return quantize(tiny_llama(), cfg, forward_loop)


def golden_buffers(env, case, mine):
    """Stock buffers from the golden file, in the engine arm's dtypes / shapes (keys checked by the caller)."""
    b = quantizer_buffers(mine)
    return {k: as_tensor(v, b[k]) if k in b else v for k, v in stored(env, case, "buf").items()}, b


def record_model(case, stock, ids_logits=None):
    for k, v in quantizer_buffers(stock).items():
        record(case, "buf", k, _np(v))
    for n, p in stock.named_parameters():
        record(case, "par", n, _np(spread(p)))


def tiny_llama(seed=0):
    from transformers import LlamaConfig, LlamaForCausalLM

    cfg = LlamaConfig(hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=2, vocab_size=256, max_position_embeddings=128, tie_word_embeddings=False)
    torch.manual_seed(seed)
    return LlamaForCausalLM(cfg).to(device="cuda", dtype=torch.bfloat16).eval()


def calib_batches(n=4, b=2, t=48, seed=1):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 256, (b, t), generator=g).cuda() for _ in range(n)]


def forward_loop(model):
    for ids in calib_batches():
        model(ids)


def quantizer_buffers(model):
    out = {}
    for name, m in model.named_modules():
        if type(m).__name__ in ("TensorQuantizer", "StaticBlockScaleQuantizer"):
            for b in ("_amax", "_global_amax", "_pre_quant_scale"):
                t = getattr(m, b, None)
                if isinstance(t, torch.Tensor):
                    out[f"{name}.{b}"] = t.detach().clone()
    return out


def run_pair(env, preset_name, algorithm=None, mutate=None):
    """-> (stock model, b200 model, stats of the b200 arm).  Without the reference: (None, mirror model, {})."""
    if not env.live:
        assert mutate is None
        return None, mirror_quantize(preset_name, algorithm), {}
    mtq, backend = env
    base = tiny_llama()
    cfg = copy.deepcopy(getattr(mtq, preset_name))
    if algorithm is not None:
        cfg["algorithm"] = algorithm
    if mutate is not None:
        mutate(cfg)
    backend.uninstall()
    stock = mtq.quantize(copy.deepcopy(base), copy.deepcopy(cfg), forward_loop)
    backend.install()
    backend.stats.clear()
    try:
        mine = mtq.quantize(copy.deepcopy(base), backend.with_b200_backend(cfg), forward_loop)
        st = dict(backend.stats)
    finally:
        backend.uninstall()
    record_model(preset_name + (f"@{algorithm}" if algorithm else ""), stock)
    return stock, mine, st


def case_buffers(env, stock, mine, what):
    """(stock buffers, engine buffers): the stock side from the model, or from the golden file."""
    if env.live:
        return quantizer_buffers(stock), quantizer_buffers(mine)
    return golden_buffers(env, what, mine)


def case_params(env, stock, mine, what):
    """[(name, stock param, engine param)]; without the reference on the stored spread sample."""
    if env.live:
        out = []
        for (n0, p0), (n1, p1) in zip(stock.named_parameters(), mine.named_parameters()):
            assert n0 == n1, (n0, n1)
            out.append((n0, p0, p1))
        return out
    ref = stored(env, what, "par")
    mp = dict(mine.named_parameters())
    assert ref.keys() == mp.keys(), sorted(set(ref) ^ set(mp))[:8]
    return [(n, as_tensor(ref[n], spread(mp[n])), spread(mp[n])) for n in ref]


def assert_buffers_equal(env, stock, mine, what):
    a, b = case_buffers(env, stock, mine, what)
    assert a.keys() == b.keys(), (what, sorted(set(a) ^ set(b))[:8])
    assert len(a) > 0 or "MX" in what, what              # MX formats keep no amax state
    bad = [k for k in a if a[k].shape != b[k].shape or a[k].dtype != b[k].dtype or not torch.equal(a[k], b[k])]
    assert not bad, (what, len(bad), bad[:6],
                     [(a[k].flatten()[:3].tolist(), b[k].flatten()[:3].tolist()) for k in bad[:3]])
    return len(a)


def mismatch_stats(ref, got):
    ref, got = ref.float(), got.float()
    zero = (ref == 0) & (got == 0)
    diff = (ref != got) & ~zero
    r, g_ = ref[diff].abs(), got[diff].abs()
    hi, lo = torch.maximum(r, g_), torch.minimum(r, g_)
    bounded = bool(((lo == 0) | (hi / lo <= 2.05)).all())
    return int(diff.sum()), bounded


def _same_to_1ulp(a, b):
    """fp32 equality up to one unit in the last place."""
    ai, bi = a.contiguous().view(torch.int32).long(), b.contiguous().view(torch.int32).long()
    return (ai - bi).abs() <= 1


def compare_outputs(env, stock, mine, exact, what):
    """Logits of both quantized models on a fresh batch (each arm through its own kernels)."""
    mtq, backend = env
    ids = calib_batches(n=1, seed=7)[0]
    with torch.no_grad():
        if env.live:
            y0 = stock(ids).logits
            record(what, "logits", "y", _np(y0))
            backend.install()
            try:
                y1 = mine(ids).logits
            finally:
                backend.uninstall()
        else:
            y1 = mine(ids).logits
            y0 = as_tensor(stored(env, what, "logits")["y"], y1)
    if exact:
        assert torch.equal(y0, y1), (what, float((y0.float() - y1.float()).abs().max()))
        return 0.0
    # NVFP4 arms differ by exact-tie roundings of a few % of the elements (one E2M1 step each, see
    # per_quantizer_outputs); through two random-init layers that is a ~10 % relative logit difference -- the
    # parity statement is the per-quantizer one, this only guards against gross divergence
    rel = float((y0.float() - y1.float()).norm() / y0.float().norm())
    assert rel < 0.3, (what, rel)
    return rel


def per_quantizer_outputs(env, stock, mine, exact, what):
    """Feed every enabled quantizer of both arms the same fresh tensor (its own weight for weight quantizers).
    Without the reference: the stored stock outputs (seeded spread sample), quantizers in the stored order."""
    if not env.live:
        return per_quantizer_outputs_golden(env, mine, exact, what)
    mtq, backend = env
    mods0, mods1 = dict(stock.named_modules()), dict(mine.named_modules())
    names = []
    g = torch.Generator(device="cuda").manual_seed(3)
    n_total = n_bad = 0
    for name, q0 in mods0.items():
        if type(q0).__name__ not in ("TensorQuantizer", "StaticBlockScaleQuantizer") or not q0.is_enabled:
            continue
        q1 = mods1[name]
        qname = name
        while qname.rsplit(".", 1)[-1].isdigit():          # a member of a SequentialQuantizer: "...weight_quantizer.0"
            qname = qname.rsplit(".", 1)[0]
        parent = mods0[qname.rsplit(".", 1)[0]]
        if qname.endswith("weight_quantizer"):
            x = parent.weight.detach()
        else:
            x = torch.randn(2, 48, parent.in_features, device="cuda", generator=g).to(torch.bfloat16) * 0.7
        with torch.no_grad():
            y0 = q0(x)
            backend.install()
            try:
                y1 = q1(x)
            finally:
                backend.uninstall()
        assert y0.shape == y1.shape and y0.dtype == y1.dtype, (what, name)
        names.append(name)
        record(what, "q", name, _np(spread(y0)))
        n, bounded = mismatch_stats(y0, y1)
        n_total += y0.numel()
        n_bad += n
        if exact:
            assert n == 0, (what, name, n)
        else:
            # NVFP4 vs the reference's Triton kernels: exact E2M1 / E4M3 rounding ties only (every mismatch within
            # one code step).  5 % like tests/test_gpu_vs_reference_triton.py: torch evaluates the global scale
            # `amax / (6 * 448)` on the GPU as a reciprocal multiply (one ulp off the IEEE value this engine uses),
            # which moves the tie set of 8-bit-mantissa data
            assert bounded and n <= 0.05 * y0.numel(), (what, name, n, y0.numel())
    assert n_total > 0
    record(what, "qnames", "order", np.array(names))
    return n_bad, n_total


def per_quantizer_outputs_golden(env, mine, exact, what):
    mods1 = dict(mine.named_modules())
    ref = stored(env, what, "q")
    g = torch.Generator(device="cuda").manual_seed(3)
    n_total = n_bad = 0
    for name in [str(n) for n in stored(env, what, "qnames")["order"]]:
        q1 = mods1[name]
        assert q1.is_enabled, (what, name)
        qname = name
        while qname.rsplit(".", 1)[-1].isdigit():
            qname = qname.rsplit(".", 1)[0]
        parent = mods1[qname.rsplit(".", 1)[0]]
        if qname.endswith("weight_quantizer"):
            x = parent.weight.detach()
        else:
            x = torch.randn(2, 48, parent.in_features, device="cuda", generator=g).to(torch.bfloat16) * 0.7
        with torch.no_grad():
            y1 = spread(q1(x))
        y0 = as_tensor(ref[name], y1)
        n, bounded = mismatch_stats(y0, y1)
        n_total += y0.numel()
        n_bad += n
        if exact:
            assert n == 0, (what, name, n)
        else:
            assert bounded and n <= 0.05 * y0.numel(), (what, name, n, y0.numel())
    assert n_total > 0
    return n_bad, n_total


# --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("preset,exact", [("INT8_DEFAULT_CFG", True), ("FP8_DEFAULT_CFG", True),
                                          ("INT4_BLOCKWISE_WEIGHT_ONLY_CFG", True), ("NVFP4_DEFAULT_CFG", False),
                                          ("FP8_PER_CHANNEL_PER_TOKEN_CFG", True), ("MXFP8_DEFAULT_CFG", True)])
def test_max_calibration_presets(env, preset, exact):
    stock, mine, st = run_pair(env, preset)
    n = assert_buffers_equal(env, stock, mine, preset)
    if env.live and preset not in ("INT4_BLOCKWISE_WEIGHT_ONLY_CFG", "MXFP8_DEFAULT_CFG", "FP8_PER_CHANNEL_PER_TOKEN_CFG"):
        assert st.get("calib.max", 0) > 0, st            # activations calibrated through the b200 collect kernel
    if env.live:
        env[1].stats.clear()
    bad, tot = per_quantizer_outputs(env, stock, mine, exact, preset)
    rel = compare_outputs(env, stock, mine, exact, preset)
    if env.live:
        assert env[1].stats.get("entrypoint", 0) > 0, dict(env[1].stats)     # fake quant ran through the b200 backend
        st["forward"] = dict(env[1].stats)
    REPORT[preset] = {"buffers_equal": n, "fake_quant_mismatch": [bad, tot], "logit_rel_diff": rel, "stats": st}


def test_int4_awq_lite(env):
    """awq_lite (model_calib.py:1395-1722) with the INT4 block-128 weight fake quant on this engine: the loss per
    alpha, hence best_alpha and the folded pre_quant_scale, must come out the same.  Without the reference the engine
    arm is the quantize() mirror, whose act_scale is one column kernel instead of ATen's reduction: the smoothed
    weights agree to one bf16 ulp (the tolerance of test_mirror_quantize_matches_reference[INT4_AWQ_CFG]), so the
    outputs are held to the rounding-tie bar instead of bit equality."""
    stock, mine, st = run_pair(env, "INT4_AWQ_CFG")
    n = assert_buffers_equal(env, stock, mine, "INT4_AWQ_CFG")
    pqs = [k for k in quantizer_buffers(mine) if k.endswith("_pre_quant_scale")]
    assert pqs, "awq_lite produced no pre_quant_scale"
    # the smoothed weights themselves
    for n0, p0, p1 in case_params(env, stock, mine, "INT4_AWQ_CFG"):
        if env.live:
            assert torch.equal(p0, p1), n0
        else:
            assert torch.allclose(p0.float(), p1.float(), rtol=2.0 ** -6, atol=1e-6), n0
    bad, tot = per_quantizer_outputs(env, stock, mine, env.live, "INT4_AWQ_CFG")
    rel = compare_outputs(env, stock, mine, env.live, "INT4_AWQ_CFG")
    REPORT["INT4_AWQ_CFG"] = {"buffers_equal": n, "pre_quant_scales": len(pqs), "fake_quant_mismatch": [bad, tot],
                              "logit_rel_diff": rel, "stats": st}


def test_int8_smoothquant(env):
    stock, mine, st = run_pair(env, "INT8_SMOOTHQUANT_CFG")
    n = assert_buffers_equal(env, stock, mine, "INT8_SMOOTHQUANT_CFG")
    for n0, p0, p1 in case_params(env, stock, mine, "INT8_SMOOTHQUANT_CFG"):
        assert torch.equal(p0, p1), n0
    rel = compare_outputs(env, stock, mine, True, "INT8_SMOOTHQUANT_CFG")
    REPORT["INT8_SMOOTHQUANT_CFG"] = {"buffers_equal": n, "logit_rel_diff": rel, "stats": st}


def test_nvfp4_static_weights_max(env):
    """Static NVFP4 weights (per-block amax + shared global amax of q/k/v and gate/up,
    utils/shared_input.py:314-346) after plain max calibration: per-block ``_amax`` and the tied ``_global_amax``
    are exact; fake quant goes through the rebound ``static_blockwise_fp4_fake_quant``."""
    stock, mine, st = run_pair(env, "NVFP4_W4A4_WEIGHT_MSE_FP8_SWEEP_CFG", algorithm="max")
    n = assert_buffers_equal(env, stock, mine, "NVFP4_W4A4_WEIGHT_MSE_FP8_SWEEP_CFG@max")
    mods = dict(mine.named_modules())
    attn = mods["model.layers.0.self_attn"]
    g = [getattr(attn, p).weight_quantizer._global_amax for p in ("q_proj", "k_proj", "v_proj")]
    assert torch.equal(g[0], g[1]) and torch.equal(g[1], g[2])
    if env.live:
        env[1].stats.clear()
    bad, tot = per_quantizer_outputs(env, stock, mine, False, "NVFP4_W4A4_WEIGHT_MSE_FP8_SWEEP_CFG@max")
    rel = compare_outputs(env, stock, mine, False, "NVFP4_W4A4_WEIGHT_MSE_FP8_SWEEP_CFG@max")
    if env.live:
        assert env[1].stats.get("fn.static_blockwise_fp4_fake_quant", 0) > 0, dict(env[1].stats)
        st["forward"] = dict(env[1].stats)
    REPORT["nvfp4_static_max"] = {"buffers_equal": n, "fake_quant_mismatch": [bad, tot], "logit_rel_diff": rel,
                                  "stats": st}


def test_nvfp4_static_mse_fp8_sweep(env):
    """mse_calibrate(fp8_scale_sweep=True): stock = the reference's Triton sweep, b200 = the registered factory
    (``_register_fp8_sweep_calibrator``) running ``b200q_nvfp4_fp8_scale_sweep``.  The winner is an argmin over 126
    fp32 losses summed in a different order: >= 99 % identical per-block winners, everything else bit-equal.
    ``best_amax = global_amax * c`` with c = e4m3 / 448: the reference builds c with torch on the GPU (a multiply by
    fl(1/448)), this engine with an IEEE division -- the same winner can differ in the last bit of the fp32 amax
    (inside the north star's "fp32 amax/scale within 1 ulp"); adjacent candidates are >= 6 % apart."""
    stock, mine, st = run_pair(env, "NVFP4_W4A4_WEIGHT_MSE_FP8_SWEEP_CFG")
    assert not env.live or st.get("calib.fp8_sweep", 0) > 0, st
    a, b = case_buffers(env, stock, mine, "NVFP4_W4A4_WEIGHT_MSE_FP8_SWEEP_CFG")
    assert a.keys() == b.keys()
    same = total = bitsame = 0
    for k in a:
        if k.endswith("weight_quantizer._amax"):
            assert a[k].shape == b[k].shape and a[k].dtype == b[k].dtype == torch.float32, k
            same += int(_same_to_1ulp(a[k], b[k]).sum())
            bitsame += int((a[k] == b[k]).sum())
            total += a[k].numel()
        else:
            assert torch.equal(a[k], b[k]), k
    assert total > 0 and same / total >= 0.99, (same, total)
    rel = compare_outputs(env, stock, mine, False, "NVFP4_W4A4_WEIGHT_MSE_FP8_SWEEP_CFG")
    REPORT["nvfp4_static_mse_fp8_sweep"] = {"same_block_winner": [same, total], "bit_identical_amax": bitsame,
                                            "logit_rel_diff": rel, "stats": st}


@pytest.mark.parametrize("preset", ["INT8_DEFAULT_CFG", "FP8_DEFAULT_CFG", "INT4_BLOCKWISE_WEIGHT_ONLY_CFG"])
def test_mse_calibrate_multiplier_search(env, preset):
    """mse_calibrate (model_calib.py:733-827) without the FP8 sweep: the 39-step multiplier search of every weight
    amax (per-channel INT8 rows, per-tensor FP8, INT4 block-128 rows).  Stock = the reference's MseCalibrator
    (39 x fake quant through its CUDA extension + ATen reductions); b200 = one sweep kernel per weight.  The
    losses are fp32 sums in a different order, so a winner may differ where two multipliers tie to ~1e-6:
    >= 99.5 % identical amax entries, all within one multiplier step."""
    stock, mine, st = run_pair(env, preset, algorithm="mse")
    assert not env.live or st.get("calib.mse", 0) > 0, st
    a, b = case_buffers(env, stock, mine, f"{preset}@mse")
    assert a.keys() == b.keys()
    same = total = 0
    for k in a:
        assert a[k].shape == b[k].shape and a[k].dtype == b[k].dtype, k
        if k.endswith("weight_quantizer._amax"):
            same += int((a[k] == b[k]).sum())
            total += a[k].numel()
            r = (a[k].float() / b[k].float())
            assert float(r.max()) < 1.6 and float(r.min()) > 0.6, (k, float(r.min()), float(r.max()))
        else:
            assert torch.equal(a[k], b[k]), k
    assert total > 0 and same / total >= 0.995, (same, total)
    REPORT[f"mse_{preset}"] = {"same_amax": [same, total], "stats": st}


@pytest.mark.parametrize("preset", ["FP8_DEFAULT_CFG", "NVFP4_DEFAULT_CFG", "INT4_BLOCKWISE_WEIGHT_ONLY_CFG",
                                    "FP8_2D_BLOCKWISE_WEIGHT_ONLY_CFG"])
def test_compress_packs_bit_exact(env, preset):
    """mtq.compress -> TensorQuantizer._real_quantize (:796-887) -> QTensor.quantize: packed bytes and scales.
    Without the reference: the engine arm packs each weight through this repo's ``_real_quantize`` and its bytes and
    scales must have the stored SHA-256 digests of the reference's."""
    mtq, backend = env
    case = f"compress/{preset}"
    stock, mine, _ = run_pair(env, preset)
    m1 = dict(mine.named_modules())
    if not env.live:
        meta = stored(env, case, "meta")
        assert meta, case
        for name, (shape, dtype) in ((n, (tuple(int(d) for d in v[:-1]), int(v[-1]))) for n, v in meta.items()):
            wq = m1[name].weight_quantizer
            with torch.no_grad():
                q = wq._real_quantize(m1[name].weight)
            data = q._quantized_data
            assert tuple(data.shape) == shape and data.element_size() == dtype, (name, tuple(data.shape), shape)
            assert np.array_equal(_digest(data), env.golden[f"{case}/pack/{name}"]), (name, preset)
            for b in ("_scale", "_double_scale"):
                key = f"{case}/{b}/{name}"
                s1 = getattr(wq, b, None)
                assert (key in env.golden) == (s1 is not None), (name, b)
                if s1 is not None:
                    assert np.array_equal(_digest(s1), env.golden[key]), (name, b, preset)
        REPORT[case] = {"packed_weights_equal": len(meta)}
        return
    mtq.compress(stock)
    backend.install()
    backend.stats.clear()
    try:
        mtq.compress(mine)
        st = dict(backend.stats)
    finally:
        backend.uninstall()
    key = {"FP8_DEFAULT_CFG": "qtensor.fp8_quantize", "FP8_2D_BLOCKWISE_WEIGHT_ONLY_CFG": "qtensor.fp8_quantize",
           "NVFP4_DEFAULT_CFG": "qtensor.nvfp4_quantize", "INT4_BLOCKWISE_WEIGHT_ONLY_CFG": "ext.INT4_quantize"}[preset]
    assert st.get(key, 0) > 0, st
    n = 0
    m1 = dict(mine.named_modules())
    for name, m0 in stock.named_modules():
        w0 = m0._parameters.get("weight") if hasattr(m0, "_parameters") else None
        if type(w0).__name__ != "QTensorWrapper":        # RealQuantLinear keeps the pack as its weight parameter
            continue
        w1 = m1[name]._parameters["weight"]
        assert type(w1).__name__ == "QTensorWrapper", name
        assert w0.metadata["shape"] == w1.metadata["shape"] and w0.metadata["dtype"] == w1.metadata["dtype"]
        assert w0.metadata["qtensor_class"] is w1.metadata["qtensor_class"], name      # the REFERENCE's QTensor class
        q0, q1 = w0.data, w1.data
        assert q0.shape == q1.shape and q0.dtype == q1.dtype, (name, q0.shape, q1.shape, q0.dtype, q1.dtype)
        assert torch.equal(q0.view(torch.uint8), q1.view(torch.uint8)), (name, preset)
        record(case, "meta", name, np.array([*q0.shape, q0.element_size()]))
        record(case, "pack", name, _digest(q0))
        for b in ("_scale", "_double_scale"):
            s0, s1 = getattr(m0.weight_quantizer, b, None), getattr(m1[name].weight_quantizer, b, None)
            assert (s0 is None) == (s1 is None), (name, b)
            if s0 is not None:
                assert s0.shape == s1.shape and s0.dtype == s1.dtype, (name, b, s0.shape, s1.shape, s0.dtype, s1.dtype)
                v0 = s0.view(torch.uint8) if s0.dtype == torch.float8_e4m3fn else s0
                v1 = s1.view(torch.uint8) if s1.dtype == torch.float8_e4m3fn else s1
                assert torch.equal(v0, v1), (name, b, preset)
                record(case, b, name, _digest(s0))
        n += 1
    assert n > 0, "no compressed weights found"
    REPORT[f"compress_{preset}"] = {"packed_weights_equal": n, "stats": st}


@pytest.mark.parametrize("preset,exact", [("INT8_DEFAULT_CFG", True), ("FP8_DEFAULT_CFG", True),
                                          ("NVFP4_DEFAULT_CFG", True), ("INT8_SMOOTHQUANT_CFG", True),
                                          ("INT4_AWQ_CFG", True), ("NVFP4_W4A4_WEIGHT_MSE_FP8_SWEEP_CFG", False),
                                          ("NVFP4_W4A4_WEIGHT_LOCAL_HESSIAN_CFG", False)])
def test_mirror_quantize_matches_reference(env, preset, exact):
    """The repo's own ``quantize()`` (the mirror of the reference interface) against the stock reference on the
    same tiny Llama: every linear's ``_amax`` / ``_global_amax`` / ``_pre_quant_scale`` and the smoothed weights."""
    mtq, backend = env
    import model_optimizer_b200.config as cfgs
    from model_optimizer_b200.model_quant import quantize

    case = f"mirror/{preset}"
    base = tiny_llama()
    mine = quantize(copy.deepcopy(base), copy.deepcopy(getattr(cfgs, preset)), forward_loop)
    if env.live:
        backend.uninstall()
        stock = mtq.quantize(copy.deepcopy(base), copy.deepcopy(getattr(mtq, preset)), forward_loop)
        a = {k: v for k, v in quantizer_buffers(stock).items() if "_bmm_quantizer" not in k and "softmax" not in k}
        for k, v in a.items():
            record(case, "buf", k, _np(v))
        for n, p in stock.named_parameters():
            record(case, "par", n, _np(spread(p)))
    else:
        stock = None
        a = stored(env, case, "buf")
    b = {}
    for name, m in mine.named_modules():
        if type(m).__name__ == "TensorQuantizer":
            for bn in ("_amax", "_global_amax", "_pre_quant_scale"):
                t = getattr(m, bn, None)
                if isinstance(t, torch.Tensor):
                    b[f"{name}.{bn}"] = t.detach()
    assert a.keys() == b.keys(), sorted(set(a) ^ set(b))[:10]
    if not env.live:
        a = {k: as_tensor(v, b[k]) for k, v in a.items()}
    same = total = 0
    awq = preset == "INT4_AWQ_CFG"
    for k in a:
        assert a[k].numel() == b[k].numel(), (k, a[k].shape, b[k].shape)
        assert a[k].dtype == b[k].dtype, (k, a[k].dtype, b[k].dtype)
        x, y = a[k].reshape(-1), b[k].reshape(-1)
        if awq:
            # AWQ-lite: act_scale is a mean of |x| over tokens -- ATen's reduction order in the reference, one column
            # kernel here: fp32 sums within ~1e-6, so the folded bf16 scales / smoothed weights / their amax may
            # differ by one bf16 ulp (DESIGN.md section 4 tolerance class); best_alpha must agree (checked below)
            eq = (x.float() - y.float()).abs() <= x.float().abs() * 2.0 ** -6
            assert bool(eq.all()), (preset, k, int((~eq).sum()))
        elif k.endswith("weight_quantizer._amax") and not exact:
            eq = _same_to_1ulp(x, y)                                # FP8 sweep winners (see the sweep test)
        else:
            eq = x == y
            assert bool(eq.all()), (preset, k, int((~eq).sum()), x[:3].tolist(), y[:3].tolist())
        same += int(eq.sum())
        total += eq.numel()
    # sweeps: argmin over 126 fp32 losses (Hessian: a 16 x 16 quadratic form summed in another order than tl.dot)
    assert same / total >= (0.97 if "HESSIAN" in preset else 0.99), (same, total)
    for n0, p0, p1 in case_params(env, stock, mine, case):
        if awq:
            assert torch.allclose(p0.float(), p1.float(), rtol=2.0 ** -6, atol=1e-6), n0
            # identical best_alpha <=> the scale vectors agree to rounding (a different alpha moves them by >> 1 ulp)
        else:
            assert torch.equal(p0, p1), n0                          # smoothquant folded weights
    REPORT[f"mirror_{preset}"] = {"buffers": len(a), "same_entries": [same, total]}


def test_hessian_sweep_vs_reference_triton_kernel(env):
    """``nvfp4_fp8_scale_sweep_hessian`` (kernels/quantization/gemm/nvfp4_fp8_sweep.py:235-290), the reference's own
    Triton kernel JIT-compiled on this box, against ``b200q_nvfp4_fp8_scale_sweep_hessian`` on the same weight and
    per-cin-block Hessian.  Winners may differ only where two candidates' fp32 losses are equal to ~1e-6."""
    from model_optimizer_b200 import ops

    if env.live:
        from modelopt.torch.kernels.quantization.gemm import nvfp4_fp8_scale_sweep_hessian

    g = torch.Generator(device="cuda").manual_seed(11)
    rep = {}
    for dtype in (torch.bfloat16, torch.float32):
        w = (torch.randn(384, 512, device="cuda", generator=g) * 0.05).to(dtype)
        x = torch.randn(2048, 512, device="cuda", generator=g) * (1 + 3 * torch.rand(512, device="cuda", generator=g))
        xt = x.float().T.reshape(512 // 16, 16, -1)
        hess = (xt @ xt.transpose(-1, -2)) / x.shape[0]
        gam = w.abs().max().float()
        got = ops.nvfp4_fp8_scale_sweep(w, gam.reshape(1), hessian=hess)
        if env.live:
            ref = nvfp4_fp8_scale_sweep_hessian(w.reshape(-1, 16), gam, hess, 16)
            record("hessian_sweep", "best", str(dtype), _np(ref))
        else:
            ref = as_tensor(stored(env, "hessian_sweep", "best")[str(dtype)], got)
        same = float(_same_to_1ulp(ref, got).float().mean())
        # the plain (unweighted) winner must differ from the Hessian one for a good share of the blocks
        plain = ops.nvfp4_fp8_scale_sweep(w, gam.reshape(1))
        moved = float((plain != got).float().mean())
        rep[str(dtype)] = {"same_winner": same, "differs_from_plain_mse": moved}
        assert same >= 0.985, (dtype, same)
        assert moved > 0.05, moved
    REPORT["hessian_sweep_vs_triton"] = rep


def test_zz_write_report():
    if GOLDEN_OUT and RECORD:
        from oracle import golden

        os.makedirs(GOLDEN_OUT, exist_ok=True)
        golden.save(GOLDEN, RECORD, GOLDEN_OUT)
    out = os.path.join(ROOT, "gpurun_out")
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "modelopt_dropin.json"), "w") as f:
        json.dump(REPORT, f, indent=1, default=str)

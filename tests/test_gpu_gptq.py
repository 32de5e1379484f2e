"""GPTQ on the GPU: the b200q_gptq_block kernel bit for bit against the C oracle (tools/gptq_oracle.c) for every covered
format, block width, row count and amax dtype, with zero rows, dead columns, tiny / huge diagonals, rounding ties and
NaN / inf weights; the kernel path of the whole update bit for bit against the composed reference loop through the
engine's quantizer; and, where the reference is installed, the engine's gptq against the stock reference's and the
drop-in's layerwise GPTQ against stock."""

import copy

import numpy as np
import pytest
import torch

from tools import gptq_oracle as orc

pytestmark = pytest.mark.gpu

ADT = {"bf16": torch.bfloat16, "f16": torch.float16, "f32": torch.float32}


def _same(a, b):
    a = np.asarray(a, dtype=np.float32)
    b = np.asarray(b, dtype=np.float32)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def _u_factor(nb, g, kind="random"):
    """An upper Cholesky factor of a damped inverse Hessian (as compute_hessian_inverse makes it), or a variant."""
    x = torch.randn(4 * nb, nb, generator=g, dtype=torch.float64)
    h = x.T @ x / (4 * nb) + 0.01 * torch.eye(nb, dtype=torch.float64)
    u = torch.linalg.cholesky(torch.cholesky_inverse(torch.linalg.cholesky(h)), upper=True).float()
    if kind == "dead":                       # a dead column: zeroed Hessian row / column, diagonal 1
        u[3, :] = 0
        u[:, 3] = 0
        u[3, 3] = 1
    elif kind == "tiny":
        u = u * 1e-30
    elif kind == "huge":
        u = u * 1e30
    return u


def _weights(rows, nb, g, fmt, case):
    w = torch.randn(rows, nb, generator=g) * 0.05
    if case == "zero_rows" and rows > 1:
        w[::2] = 0
    elif case == "nonfinite":
        w[0, 1] = float("nan")
        if rows > 1:
            w[rows // 2, nb // 2] = float("inf")
            w[rows - 1, nb - 1] = float("-inf")
    return w


def _quant_args(fmt, rows, in_f, col0, g, adt, layout):
    """(kernel kwargs, oracle kwargs) for one format / amax layout."""
    if fmt == orc.FMT_NVFP4_DYNAMIC:
        amax = torch.tensor([0.2], dtype=adt)
        return {"amax": amax.cuda()}, {"amax": amax.float().numpy()}
    if fmt == orc.FMT_NVFP4_STATIC:
        amax = (torch.rand(rows * in_f // 16, generator=g) * 0.2 + 0.01)
        amax[:3] = 0                                   # a zero block scale
        ga = torch.tensor(0.21)
        kw = {"amax": amax.cuda(), "amax_row_stride": in_f // 16, "amax_col_block": 16, "global_amax": ga.cuda()}
        return kw, {"amax": amax.numpy(), "amax_row_stride": in_f // 16, "amax_col_block": 16,
                    "global_amax": float(ga)}
    if layout == "tensor":
        amax, rs, cb = torch.tensor([0.11]), 0, orc.PER_TENSOR_COL_BLOCK
    elif layout == "row":
        amax, rs, cb = torch.rand(rows, 1, generator=g) * 0.2 + 1e-9, 1, orc.PER_TENSOR_COL_BLOCK
        amax[0] = 0
    else:                                              # per (row, 32-column block)
        amax, rs, cb = torch.rand(rows * in_f // 32, generator=g) * 0.2, in_f // 32, 32
    amax = amax.to(adt)
    kw = {"amax": amax.cuda(), "amax_row_stride": rs, "amax_col_block": cb}
    okw = {"amax": amax.float().numpy(), "amax_row_stride": rs, "amax_col_block": cb}
    if fmt == orc.FMT_INT:
        kw.update(num_bits=4 if layout == "block" else 8, narrow_range=layout == "row")
        okw.update(num_bits=4 if layout == "block" else 8, narrow_range=layout == "row")
    return kw, okw


TIE_GLOBAL_AMAX = 2688 * 2.0 ** -14     # NVFP4: per-tensor scale 2^-14
TIE_BLOCK_MAX = 0.09375                  # NVFP4: a 16-element block with this |x| max gets the block scale 2^-6


def _make_ties(fmt, layout, w, u, kw, okw, g):
    """Put column 16k of every 16-column block exactly on rounding ties of the scale in use, and keep it (and, for
    NVFP4, column 16k + 15, which sets the block amax) unperturbed by earlier columns: zero U above those columns.
    INT: amax = bound * 2^-10 (scale 2^10), x = (k + 1/2) * 2^-10.  FP8: amax = 448 * 2^-10, x on midpoints of the
    E4M3 grid.  NVFP4: block scale 2^-6 (static: block amax 0.09375 with global amax 0.1640625; dynamic: the same
    global amax and a block max of 0.09375), x on the E2M1 decision boundaries."""
    rows, nb = w.shape
    cols = list(range(0, nb, 16))
    keep = cols + ([c + 15 for c in cols] if fmt in (orc.FMT_NVFP4_STATIC, orc.FMT_NVFP4_DYNAMIC) else [])
    for c in keep:
        u[:c, c] = 0
    sign = torch.where(torch.rand(rows, len(cols), generator=g) < 0.5, -1.0, 1.0)
    if fmt == orc.FMT_INT:
        bound = (1 << (kw.get("num_bits", 8) - 1)) - 1
        val = bound * 2.0 ** -10
        k = torch.randint(-bound, bound, (rows, len(cols)), generator=g).float()
        w[:, cols] = (k + 0.5) * 2.0 ** -10
    elif fmt == orc.FMT_FP8:
        val = 448 * 2.0 ** -10
        j = torch.randint(0, 8, (rows, len(cols)), generator=g).float()
        e = torch.randint(-3, 4, (rows, len(cols)), generator=g).float()
        w[:, cols] = sign * (1 + (2 * j + 1) / 16) * 2.0 ** e * 2.0 ** -10
    else:
        bnd = torch.tensor([0.25, 0.75, 1.25, 1.75, 2.5, 3.5, 5.0])
        w[:, keep] = w[:, keep].clamp(-0.05, 0.05)
        w[:, cols] = sign * bnd[torch.randint(0, 7, (rows, len(cols)), generator=g)] * 2.0 ** -6
        w[:, [c + 15 for c in cols]] = TIE_BLOCK_MAX
        val = TIE_BLOCK_MAX if fmt == orc.FMT_NVFP4_STATIC else TIE_GLOBAL_AMAX
        if fmt == orc.FMT_NVFP4_STATIC:
            kw["global_amax"] = torch.tensor(TIE_GLOBAL_AMAX, device="cuda")
            okw["global_amax"] = TIE_GLOBAL_AMAX
    kw["amax"] = torch.full_like(kw["amax"], val)
    okw["amax"] = kw["amax"].float().cpu().numpy()
    assert (kw["amax"].float() == val).all()                      # representable in the amax dtype


FORMATS = [(orc.FMT_INT, "tensor"), (orc.FMT_INT, "row"), (orc.FMT_INT, "block"), (orc.FMT_FP8, "tensor"),
           (orc.FMT_FP8, "row"), (orc.FMT_NVFP4_STATIC, "block"), (orc.FMT_NVFP4_DYNAMIC, "tensor")]


@pytest.mark.parametrize("fmt,layout", FORMATS)
@pytest.mark.parametrize("nb", [16, 32, 64, 128])
@pytest.mark.parametrize("rows", [1, 7, 1027])
def test_kernel_vs_oracle(fmt, layout, nb, rows):
    from model_optimizer_b200 import ops

    g = torch.Generator().manual_seed(nb * 1000 + rows + 17 * fmt)
    in_f, col0 = 2 * nb if nb <= 64 else nb, nb if nb <= 64 else 0       # a second block: amax indexing by col0
    cases = [("random", "random", "f32"), ("zero_rows", "dead", "bf16"), ("ties", "random", "f16"),
             ("ties", "random", "f32"), ("random", "tiny", "f32"), ("random", "huge", "bf16"), ("nonfinite", "random", "f32")]
    for wcase, ukind, ad in cases:
        adt = ADT[ad]
        if fmt == orc.FMT_NVFP4_STATIC and ad != "f32":
            continue                                   # promoted static NVFP4 keeps its block amax in fp32
        w = _weights(rows, nb, g, fmt, wcase)
        u = _u_factor(nb, g, ukind)
        kw, okw = _quant_args(fmt, rows, in_f, col0, g, adt, layout)
        if wcase == "ties":
            _make_ties(fmt, layout, w, u, kw, okw, g)
        full = torch.zeros(rows, in_f)                 # the block lives at columns [col0, col0 + nb) of a wider matrix
        full[:, col0:col0 + nb] = w
        wd = full.cuda()
        ud = torch.zeros(nb, nb + 5)                   # a U block with a leading dimension; lower triangle garbage
        ud[:, :nb] = u + torch.tril(torch.full((nb, nb), 7.0), -1)
        ud = ud.cuda()
        e = ops.gptq_block_update(wd[:, col0:col0 + nb], ud[:, :nb], fmt, col0=col0, **kw)
        want_w, want_e = orc.gptq_block(w.numpy(), u.numpy(), fmt, col0=col0, **okw)
        got_w = wd[:, col0:col0 + nb].cpu().numpy()
        ok_w, ok_e = _same(got_w, want_w), _same(e.cpu().numpy(), want_e)
        assert ok_w.all() and ok_e.all(), (wcase, ukind, ad, int((~ok_w).sum()), int((~ok_e).sum()))
        assert (wd[:, :col0] == 0).all() and (wd[:, col0 + nb:] == 0).all()    # nothing outside the block


def _quantizer(kind, w):
    """A calibrated engine weight quantizer for ``w`` (max calibration on the weight itself)."""
    from model_optimizer_b200.config import QuantizerAttributeConfig
    from model_optimizer_b200.nn import TensorQuantizer

    cfgs = {"int8_row": {"num_bits": 8, "axis": 0}, "fp8": {"num_bits": (4, 3), "axis": None},
            "int4_b128": {"num_bits": 4, "block_sizes": {-1: 128, "type": "static"}},
            "int4_b16": {"num_bits": 4, "block_sizes": {-1: 16, "type": "static"}},
            "nvfp4_dyn": {"num_bits": (2, 1), "block_sizes": {-1: 16, "type": "dynamic", "scale_bits": (4, 3)}},
            "nvfp4_static": {"num_bits": (2, 1), "block_sizes": {-1: 16, "type": "static", "scale_bits": (4, 3)}}}
    q = TensorQuantizer(QuantizerAttributeConfig(**cfgs[kind])).cuda()
    q.disable_quant()
    q.enable_calib()
    q(w)
    q.load_calib_amax()
    q.disable_calib()
    q.enable_quant()
    if q.is_static_block_quant and q._amax.dtype != torch.float32:   # promoted static blocks keep fp32 amax
        blocks = q._amax.float()
        delattr(q, "_amax")
        q.amax = blocks
    if q.is_nvfp4_static:
        from model_optimizer_b200 import ops

        gl = torch.zeros(1, dtype=torch.float32, device=w.device)
        ops.amax_per_tensor_(gl, q._amax.contiguous())
        q.register_buffer("_global_amax", gl.reshape(()))
    return q


@pytest.mark.parametrize("kind", ["int8_row", "fp8", "int4_b128", "int4_b16", "nvfp4_dyn", "nvfp4_static"])
@pytest.mark.parametrize("block_size,in_f", [(16, 96), (128, 384), (128, 320)])
@pytest.mark.parametrize("wdt", ["bf16", "f32"])
def test_kernel_path_vs_composed_loop(kind, block_size, in_f, wdt):
    from model_optimizer_b200 import model_calib, ops

    if kind == "int4_b128" and in_f % 128:
        pytest.skip("a padded block layout takes the composed loop on both sides")
    g = torch.Generator().manual_seed(in_f + block_size)
    out_f = 48
    w0 = (torch.randn(out_f, in_f, generator=g) * 0.05).to(ADT[wdt]).cuda()
    x = torch.randn(256, in_f, generator=g).cuda()
    h, n = model_calib.update_hessian(x, torch.zeros(in_f, in_f, device="cuda"), 0)
    q = _quantizer(kind, w0)
    weight = w0.float().clone()
    h_inv = model_calib.compute_hessian_inverse(h, weight, 0.01)
    desc = ops.gptq_quantizer_desc(q, weight.shape)
    assert desc is not None
    a = weight.clone()
    ops.gptq_blockwise_update(a, h_inv, block_size, q, desc=desc)
    b = weight.clone()
    model_calib.gptq_blockwise_update_composed(b, h_inv, block_size, q)
    same = _same(a.cpu().numpy(), b.cpu().numpy())
    assert same.all(), int((~same).sum())
    assert not torch.equal(a, weight)


def test_out_of_scope_quantizers_take_the_composed_loop():
    from model_optimizer_b200 import model_calib, ops
    from model_optimizer_b200.config import QuantizerAttributeConfig
    from model_optimizer_b200.nn import TensorQuantizer

    w = torch.randn(32, 64, device="cuda") * 0.1
    mx = TensorQuantizer(QuantizerAttributeConfig(num_bits=(4, 3), block_sizes={-1: 32, "type": "dynamic",
                                                                                 "scale_bits": (8, 0)})).cuda()
    dyn = TensorQuantizer(QuantizerAttributeConfig(num_bits=8, axis=None, type="dynamic")).cuda()
    for q in (mx, dyn):
        assert ops.gptq_quantizer_desc(q, w.shape) is None
        h_inv = torch.eye(64, device="cuda")
        a = w.clone()
        assert model_calib.gptq_blockwise_update(a, h_inv, 32, q) is False
        b = w.clone()
        model_calib.gptq_blockwise_update_composed(b, h_inv, 32, q)
        assert torch.equal(a, b)


# ---- the engine's gptq and the drop-in against the stock reference ---------------------------------------------
def _tiny_llama(seed=0):
    from transformers import LlamaConfig, LlamaForCausalLM

    cfg = LlamaConfig(hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=2, vocab_size=256, max_position_embeddings=128, tie_word_embeddings=False)
    torch.manual_seed(seed)
    return LlamaForCausalLM(cfg).to(device="cuda", dtype=torch.bfloat16).eval()


def _forward_loop(model):
    g = torch.Generator().manual_seed(1)
    for _ in range(4):
        model(torch.randint(0, 256, (2, 48), generator=g).cuda())


def _linear_hessians(model):
    """2 X X^T / n per linear, from the unquantized tiny model (the weight used for the error metric)."""
    hs, hooks = {}, []
    for n, m in model.named_modules():
        if isinstance(m, torch.nn.Linear) and "lm_head" not in n:
            def hook(mod, args, n=n):
                x = args[0].reshape(-1, args[0].shape[-1]).float()
                h, c = hs.get(n, (0, 0))
                hs[n] = (h + 2 * x.T @ x, c + x.shape[0])
            hooks.append(m.register_forward_pre_hook(hook))
    with torch.no_grad():
        _forward_loop(model)
    for h in hooks:
        h.remove()
    return {n: h / c for n, (h, c) in hs.items()}


def _rel_err(w, w0, h):
    w, w0 = w.detach(), w0.detach()
    d = w.float() - w0.float()
    return float((d @ h * d).mean() / ((w0.float() @ h * w0.float()).mean() + 1e-6))


EXACT = ["INT8_DEFAULT_CFG", "FP8_DEFAULT_CFG", "INT4_BLOCKWISE_WEIGHT_ONLY_CFG"]
NVFP4 = ["NVFP4_DEFAULT_CFG", "NVFP4_STATIC", "NVFP4_W4A16", "NVFP4_STATIC_W4A16"]
PRESETS = EXACT + NVFP4


def _edit(cfg, preset):
    """NVFP4 variants of NVFP4_DEFAULT_CFG: static weight blocks, and / or input quantizers off (weight-only)."""
    for e in cfg["quant_cfg"]:
        if isinstance(e, dict) and e.get("quantizer_name") == "*weight_quantizer" and isinstance(e.get("cfg"), dict) \
                and "STATIC" in preset:
            e["cfg"]["block_sizes"] = dict(e["cfg"]["block_sizes"], type="static")
    if "W4A16" in preset:
        cfg["quant_cfg"].append({"quantizer_name": "*input_quantizer", "enable": False})
    return cfg


def _stock_cfg(mtq, preset, layerwise=False):
    cfg = copy.deepcopy(mtq.NVFP4_DEFAULT_CFG if preset in NVFP4 else getattr(mtq, preset))
    cfg = _edit(cfg, preset)
    cfg["algorithm"] = {"method": "gptq", **({"layerwise": {"enable": True}} if layerwise else {})}
    return cfg


def _mirror_cfg(preset):
    import model_optimizer_b200.config as cfgs

    cfg = _edit(copy.deepcopy(cfgs.NVFP4_DEFAULT_CFG if preset in NVFP4 else getattr(cfgs, preset)), preset)
    cfg["algorithm"] = {"method": "gptq"}
    return cfg


E2M1_RATIOS = (4 / 3, 1.5, 2.0)   # the ratios of adjacent non-zero E2M1 levels 0.5, 1, 1.5, 2, 3, 4, 6


def _check_rows(name, mine, stock):
    """The NVFP4 tie rules (DESIGN §4) per row: identical, or the first difference is one step -- one E2M1 step under
    the same block scale (same sign; ratio 4/3, 3/2 or 2, or zero against the smallest level), or the same E2M1 level
    under block scales one E4M3 step apart (ratio at most 1 + 1/8).  The weights are stored in bf16: ratios to 1 %."""
    a, b = mine.detach().float().cpu(), stock.detach().float().cpu()
    diff = a != b
    bad = []
    for r in diff.any(dim=1).nonzero().flatten().tolist():
        c = int(diff[r].nonzero()[0])
        x, y = float(a[r, c]), float(b[r, c])
        lo, hi = sorted((abs(x), abs(y)))
        blk = float(torch.maximum(a[r, c // 16 * 16:c // 16 * 16 + 16].abs().max(),
                                  b[r, c // 16 * 16:c // 16 * 16 + 16].abs().max()))
        if x * y < 0:
            ok = False
        elif lo == 0:
            ok = hi <= blk / 12 * 1.02                    # 0.5 s against 0, with the block max at most 6 s
        else:
            ok = any(abs(hi / lo - k) <= 0.01 * k for k in E2M1_RATIOS) or hi / lo <= 1.125 * 1.01
        if not ok:
            bad.append((r, c, x, y))
    assert not bad, (name, len(bad), bad[:4])
    return int(diff.any(dim=1).sum())


def _compare(preset, mine, stock, base, row_rule_layers=(0,)):
    """INT / FP8: weights and amax bit-identical.  NVFP4: amax bit-identical, the per-row rule on the first decoder
    layer of a weight-only config (its inputs are the embeddings through one RMSNorm on both sides, so its Hessians
    agree), and the Hessian-weighted relative errors of the two runs on every module."""
    hs = _linear_hessians(base)
    sm = dict(stock.named_modules())
    bm = dict(base.named_modules())
    n_cmp, spread = 0, {}
    for n, m in mine.named_modules():
        if n not in hs or not hasattr(m, "weight_quantizer"):
            continue
        s = sm[n]
        if preset in EXACT:
            assert torch.equal(m.weight, s.weight), n
            assert torch.equal(m.weight_quantizer._amax.float(), s.weight_quantizer._amax.float()), n
        else:
            assert torch.equal(m.weight_quantizer._amax.float(), s.weight_quantizer._amax.float()), n
            if "W4A16" in preset and any(f"layers.{k}." in n for k in row_rule_layers):
                _check_rows(n, m.weight, s.weight)
            em, es = _rel_err(m.weight, bm[n].weight, hs[n]), _rel_err(s.weight, bm[n].weight, hs[n])
            spread[n] = abs(em - es) / es
        n_cmp += 1
    assert n_cmp > 0
    # One tie rounded differently (the stock side quantizes NVFP4 with Triton) changes every later column of the row,
    # and where input quantizers are on, the Hessians differ too.  Measured spread of the relative errors on this
    # model: up to 1.4 % in the first layer, up to 4.1 % in the second.
    assert all(v <= 0.05 for v in spread.values()), sorted(spread.items(), key=lambda kv: -kv[1])[:4]


@pytest.fixture(scope="module")
def ref():
    from baseline import ref_env

    if not ref_env.available():
        pytest.skip("the stock reference is not installed")
    mtq = ref_env.activate()
    ref_env.use_prebuilt_extensions()
    return mtq


def _n_linears(model):
    """Linear layers with an enabled weight quantizer: the modules GPTQ updates."""
    return sum(1 for m in model.modules() if isinstance(m, torch.nn.Linear) and m.weight_quantizer.is_enabled)


@pytest.mark.parametrize("preset", PRESETS)
def test_mirror_gptq_vs_stock(ref, preset):
    from model_optimizer_b200 import model_calib
    from model_optimizer_b200.model_quant import quantize

    before = model_calib.stats["gptq.kernel"]
    mine = quantize(_tiny_llama(), _mirror_cfg(preset), _forward_loop)
    assert model_calib.stats["gptq.kernel"] - before == _n_linears(mine)      # every weight took the kernel
    stock = ref.quantize(_tiny_llama(), _stock_cfg(ref, preset), _forward_loop)
    _compare(preset, mine, stock, _tiny_llama(), row_rule_layers=(0,))


@pytest.mark.parametrize("preset", ["INT4_BLOCKWISE_WEIGHT_ONLY_CFG", "NVFP4_DEFAULT_CFG", "NVFP4_STATIC"])
def test_mirror_gptq_kernel_vs_composed(monkeypatch, preset):
    """The engine's gptq with the kernel and with every quantizer forced onto the composed loop: bit-identical."""
    from model_optimizer_b200 import model_calib, ops
    from model_optimizer_b200.model_quant import quantize

    a = quantize(_tiny_llama(), _mirror_cfg(preset), _forward_loop)
    before = model_calib.stats["gptq.composed"]
    monkeypatch.setattr(ops, "gptq_quantizer_desc", lambda *args, **kw: None)
    b = quantize(_tiny_llama(), _mirror_cfg(preset), _forward_loop)
    assert model_calib.stats["gptq.composed"] - before == _n_linears(b)
    for (n, x), (_, y) in zip(a.named_parameters(), b.named_parameters()):
        assert torch.equal(x, y), n


@pytest.mark.parametrize("preset", PRESETS + ["MXFP8_DEFAULT_CFG"])
def test_dropin_layerwise_gptq_vs_stock(ref, preset):
    from model_optimizer_b200 import backend

    stock = ref.quantize(_tiny_llama(), _stock_cfg(ref, preset, layerwise=True), _forward_loop)
    backend.install()
    try:
        before = backend.stats["gptq.block"]
        mine = ref.quantize(_tiny_llama(), backend.with_b200_backend(_stock_cfg(ref, preset, layerwise=True)),
                            _forward_loop)
        ran = backend.stats["gptq.block"] - before
    finally:
        backend.uninstall()
    if preset == "MXFP8_DEFAULT_CFG":
        assert ran == 0
        for (n, a), (_, b) in zip(mine.named_parameters(), stock.named_parameters()):
            assert torch.equal(a, b), n
        return
    assert ran == _n_linears(mine)
    _compare(preset, mine, stock, _tiny_llama())


@pytest.mark.parametrize("preset", PRESETS)
def test_dropin_helper_vs_reference_loop(ref, preset):
    """Layerwise GPTQ through the drop-in with B200GPTQHelper registered for "b200", and again with the reference's
    own GPTQHelper registered instead: both quantize through the b200 entrypoint, so the weights are bit-identical.
    This checks how the helper reads the reference's quantizers (amax layout and dtype, global amax) exactly."""
    from modelopt.torch.quantization.utils import calib_utils as cu

    from model_optimizer_b200 import backend

    backend.install()
    helper = cu._GPTQ_HELPER_REGISTRY["b200"]
    try:
        before = backend.stats["gptq.block"]
        a = ref.quantize(_tiny_llama(), backend.with_b200_backend(_stock_cfg(ref, preset, layerwise=True)),
                         _forward_loop)
        assert backend.stats["gptq.block"] - before == _n_linears(a)
        cu.register_gptq_helper("b200", cu.GPTQHelper)
        before = backend.stats["gptq.block"]
        b = ref.quantize(_tiny_llama(), backend.with_b200_backend(_stock_cfg(ref, preset, layerwise=True)),
                         _forward_loop)
        assert backend.stats["gptq.block"] == before
    finally:
        cu.register_gptq_helper("b200", helper)
        backend.uninstall()
    for (n, x), (_, y) in zip(a.named_parameters(), b.named_parameters()):
        assert torch.equal(x, y), n

"""Unified-HF checkpoint export -- the step right after the hot path (SURVEY.md 8(f1)).

Mirror of ``modelopt/torch/export/unified_export_hf.py`` for dense decoder-only HF models (``LlamaForCausalLM``
layout) and every weight format the engine calibrates: FP8 per-tensor, per-channel and 2-D block, INT8 SmoothQuant and
weight-only, MXFP8, MXFP4, W4A8-MXFP4-FP8, NVFP4 dynamic / static, W4A16-NVFP4, NVFP4-AWQ, W4A8-NVFP4-FP8 and
INT4-AWQ, one format per model or mixed precision:

  * ``fuse_prequant_to_linear`` (quant_utils.py:1354-1429) -- for an NVFP4-AWQ model, the pre_quant_scale of
    down_proj (o_proj) is folded into the output rows of up_proj (v_proj) where the sizes agree;
  * ``requantize_resmooth_fused_llm_layers`` (:421-540) -- linears that read the same tensor (q/k/v, gate/up) are found
    with forward hooks on a dummy forward, then ``preprocess_linear_fusion`` (quant_utils.py:1475-1545) re-smooths
    them to ONE averaged ``pre_quant_scale`` (weights rescaled and re-calibrated), unifies the input amax and the
    per-tensor weight amax / NVFP4 global amax, and ``fuse_prequant_layernorm`` (:1442-1472) folds the shared
    pre_quant_scale into the preceding norm;
  * ``_export_quantized_weight`` (:569-800) per linear: ``weight`` (packed), ``weight_scale``, ``weight_scale_2``,
    ``input_scale`` -- every pack is one kernel of this engine (``export.py``);
  * ``postprocess_state_dict`` (quant_utils.py:1054-1110): quantizer state dropped, ``input_quantizer._pre_quant_scale``
    renamed to ``pre_quant_scale``;
  * ``hf_quant_config.json`` (quant_utils.py:1583-1700, process_layer_quant_config :680-789: one format, or
    ``MIXED_PRECISION`` with per-layer ``quantized_layers``) and ``model.safetensors``.

Pinned byte for byte against the reference's own export of the same calibrated state (tests/golden/ref_export.npz,
tests/golden/ref_export_formats*.npz).
"""

from __future__ import annotations

import json
import os
from collections import defaultdict

import torch
from torch import nn

from . import export as ex
from . import model_calib
from .nn import TensorQuantizer, is_quantized_linear

# hf_quant_config.json per-layer entries (quant_utils.py:680-770): the quant_algo string of each format, and whether
# it also carries group_size (the weight block size) and has_zero_point / pre_quant_scale; other formats are
# written under their own label
_ALGO = {ex.QUANTIZATION_FP8: ("FP8", False, False), ex.QUANTIZATION_FP8_PC_PT: ("FP8_PER_CHANNEL_PER_TOKEN", False, False),
         ex.QUANTIZATION_INT4_AWQ: ("W4A16_AWQ", True, True), ex.QUANTIZATION_INT8_WO: ("W8A16", False, False),
         ex.QUANTIZATION_INT8_SQ: ("W8A8_SQ_PER_CHANNEL", False, False), ex.QUANTIZATION_NVFP4: ("NVFP4", True, False),
         ex.QUANTIZATION_W4A16_NVFP4: ("W4A16_NVFP4", True, False), ex.QUANTIZATION_NVFP4_AWQ: ("NVFP4_AWQ", True, True),
         ex.QUANTIZATION_W4A8_NVFP4_FP8: ("W4A8_NVFP4_FP8", True, False),
         ex.QUANTIZATION_W4A8_MXFP4_FP8: ("W4A8_MXFP4_FP8", True, False), ex.QUANTIZATION_MXFP8: ("MXFP8", True, False)}
# pre_quant_scale of the second linear folded into the output rows of the first (quant_utils.py:1340-1351)
_PQS_FUSE_PAIRS = {"LlamaAttention": ("v_proj", "o_proj"), "Qwen3Attention": ("v_proj", "o_proj"),
                   "Qwen3MoeAttention": ("v_proj", "o_proj"), "LlamaMLP": ("up_proj", "down_proj"),
                   "Qwen3MLP": ("up_proj", "down_proj"), "Qwen3MoeMLP": ("up_proj", "down_proj")}


def _is_layernorm(m: nn.Module) -> bool:
    name = type(m).__name__.lower()
    return ("layernorm" in name or "rmsnorm" in name) and getattr(m, "weight", None) is not None


def _enabled(q) -> bool:
    return isinstance(q, TensorQuantizer) and q.is_enabled


# ---- shared-input discovery (unified_export_hf.py:279-349) ------------------------------------------------------
@torch.no_grad()
def collect_shared_input_modules(model: nn.Module, dummy_forward):
    """-> ({input tensor id: [linears]}, {norm output tensor id: norm}); quantizers disabled during the probe."""
    input_to_linear: dict = defaultdict(list)
    output_to_norm: dict = {}
    keep = []                                   # keep the probed tensors alive so that ids stay unique
    handles = []

    def in_hook(mod, args, out):
        if args and isinstance(args[0], torch.Tensor):
            keep.append(args[0])
            input_to_linear[id(args[0])].append(mod)

    def out_hook(mod, args, out):
        if isinstance(out, torch.Tensor):
            keep.append(out)
            output_to_norm[id(out)] = mod

    for _, m in model.named_modules():
        if _is_layernorm(m):
            handles.append(m.register_forward_hook(out_hook))
        elif is_quantized_linear(m) and (_enabled(m.input_quantizer) or _enabled(m.weight_quantizer)):
            handles.append(m.register_forward_hook(in_hook))
    qs = [q for q in model.modules() if isinstance(q, TensorQuantizer)]
    saved = [q._disabled for q in qs]
    try:
        for q in qs:
            q._disabled = True
        dummy_forward()
    finally:
        for q, d in zip(qs, saved):
            q._disabled = d
        for h in handles:
            h.remove()
    return input_to_linear, output_to_norm


# ---- fusion preprocessing (quant_utils.py:1285-1302, 1442-1545) ---------------------------------------------------
@torch.no_grad()
def _update_pre_quant_scale(module, new_pqs):
    old = module.input_quantizer._pre_quant_scale
    dtype = module.weight.dtype
    w = (module.weight.to(torch.float32) * old.to(dtype=torch.float32, device=module.weight.device)
         / new_pqs.to(dtype=torch.float32, device=module.weight.device)).to(dtype)
    module.weight.copy_(w)
    module.input_quantizer.pre_quant_scale = new_pqs
    wq = module.weight_quantizer                       # redo the weight collection
    wq.reset_amax()
    model_calib.max_calibrate(wq, lambda q: q(module.weight), distributed_sync=False)
    model_calib._finalize_static_nvfp4(module)         # promoted (fp32) state like the reference's quantizer class


@torch.no_grad()
def preprocess_linear_fusion(modules, resmooth_only=False):
    fmts = [ex.get_quantization_format(m) for m in modules]
    assert all(f == fmts[0] for f in fmts), "Modules have different quantization formats"
    iq0 = modules[0].input_quantizer
    if iq0.pre_quant_scale is not None:
        avg = torch.mean(torch.stack([m.input_quantizer.pre_quant_scale for m in modules]), dim=0)
        for m in modules:
            if not torch.equal(m.input_quantizer.pre_quant_scale, avg):
                _update_pre_quant_scale(m, avg)
    if resmooth_only:
        return
    if iq0.is_enabled and iq0.amax is not None:
        assert iq0.amax.numel() == 1, "Only support scalar input quant amax"
        amax = torch.max(torch.stack([m.input_quantizer.amax.reshape(()) for m in modules]))
        for m in modules:
            m.input_quantizer.amax = amax.reshape(m.input_quantizer.amax.shape)
    wq0 = modules[0].weight_quantizer
    if getattr(wq0, "_global_amax", None) is not None:          # static NVFP4: one global amax for the fused group
        g = torch.max(torch.stack([m.weight_quantizer._global_amax.reshape(()) for m in modules]))
        for m in modules:
            m.weight_quantizer._global_amax.copy_(g)
            m.weight_quantizer._state_gen += 1
    elif wq0.is_enabled and wq0.amax is not None and wq0.amax.numel() == 1:
        amax = torch.max(torch.stack([m.weight_quantizer.amax.reshape(()) for m in modules]))
        for m in modules:
            m.weight_quantizer.amax = amax.reshape(m.weight_quantizer.amax.shape)


@torch.no_grad()
def fuse_prequant_layernorm(norm: nn.Module, modules):
    iq = modules[0].input_quantizer
    if not hasattr(iq, "_pre_quant_scale"):
        return
    pqs = iq._pre_quant_scale.to(norm.weight.device)
    norm.weight.copy_((norm.weight * pqs).to(norm.weight.dtype))
    if getattr(norm, "bias", None) is not None:
        norm.bias.copy_(norm.bias * pqs)
    for m in modules:
        delattr(m.input_quantizer, "_pre_quant_scale")
        m.fused_with_prequant = True


@torch.no_grad()
def fuse_prequant_to_linear(model: nn.Module):
    """quant_utils.py:1354-1429 without grouped heads: where the consumer's pre_quant_scale has one entry per output
    row of the producer (o_proj after v_proj, down_proj after up_proj), scale those rows, re-collect the producer's
    weight amax and drop the consumer's pre_quant_scale.  GQA attention (fewer v_proj rows) is skipped."""
    for m in model.modules():
        pair = next((p for k, p in _PQS_FUSE_PAIRS.items() if k in type(m).__name__), None)
        if pair is None:
            continue
        into, src = m.get_submodule(pair[0]), m.get_submodule(pair[1])
        pqs = getattr(getattr(src, "input_quantizer", None), "_pre_quant_scale", None)
        if pqs is None or pqs.numel() != into.weight.shape[-2]:
            continue
        into.weight.copy_(into.weight * pqs.view(-1, 1))
        if into.bias is not None:
            into.bias.copy_(into.bias * pqs)
        wq = into.weight_quantizer
        wq.reset_amax()
        model_calib.max_calibrate(wq, lambda q: q(into.weight), distributed_sync=False)
        model_calib._finalize_static_nvfp4(into)
        delattr(src.input_quantizer, "_pre_quant_scale")
        src.input_quantizer._state_gen += 1
        src.fused_with_prequant = True


def _model_format(model: nn.Module):
    """The first quantized linear's format (quant_utils.py:593-603 on the root module)."""
    for m in model.modules():
        if is_quantized_linear(m):
            f = ex.get_quantization_format(m)
            if f is not None:
                return f
    return None


@torch.no_grad()
def requantize_resmooth_fused_llm_layers(model: nn.Module):
    device = next(model.parameters()).device
    if _model_format(model) == ex.QUANTIZATION_NVFP4_AWQ:          # unified_export_hf.py:445-446
        fuse_prequant_to_linear(model)

    def dummy():
        model(torch.ones([1, 2], dtype=torch.long, device=device))

    input_to_linear, output_to_norm = collect_shared_input_modules(model, dummy)
    fused = []
    for tid, modules in input_to_linear.items():
        fmt = ex.get_quantization_format(modules[0])
        if len(modules) > 1 and fmt not in (ex.QUANTIZATION_FP8, ex.QUANTIZATION_NONE):
            preprocess_linear_fusion(modules)
            fused.append(modules)
            if fmt is not None and "awq" in fmt and tid in output_to_norm:
                fuse_prequant_layernorm(output_to_norm[tid], modules)
    return fused


# ---- per-linear export (unified_export_hf.py:569-800) ---------------------------------------------------------------
@torch.no_grad()
def export_linear_tensors(module) -> dict:
    """{suffix: tensor} for one quantized linear, the reference's names, dtypes and shapes."""
    fmt = ex.get_quantization_format(module)
    wq, iq = module.weight_quantizer, module.input_quantizer
    w = module.weight.detach()
    out = {}
    if fmt == ex.QUANTIZATION_FP8:
        amax = wq._amax.to(torch.float32)
        wsf = ex._tdiv(amax, wq.maxbound).reshape(())                    # 0-dim: `weight / scale` stays in the weight dtype
        out["weight_scale"] = wsf
        out["weight"] = ex.to_quantized_weight(w, wsf, fmt)
        if getattr(iq, "_amax", None) is not None and iq.is_enabled:
            out["input_scale"] = ex._tdiv(iq._amax.to(torch.float32), iq.maxbound).squeeze()
        return out
    if fmt in ex._NVFP4_FORMATS:
        packed, scales, wsf2 = ex.export_nvfp4_weight(module)
        out.update(weight=packed, weight_scale=scales, weight_scale_2=wsf2.reshape(()))
    elif fmt == ex.QUANTIZATION_INT4_AWQ:
        amax = wq.export_amax()                                            # [out, in / block]
        wsf = ex._tdiv(amax.float(), wq.maxbound).reshape(w.shape[0], -1)
        out.update(weight=ex.pack_int4_in_uint8(w, wsf), weight_scale=wsf)
    elif fmt in (ex.QUANTIZATION_FP8_PC_PT, *ex._INT8_FORMATS):
        wsf = ex.get_scaling_factor(wq).reshape(-1)                        # [out] fp32: the quotient is fp32
        out.update(weight=ex.to_quantized_weight(w, wsf, fmt), weight_scale=wsf)
    elif fmt == ex.QUANTIZATION_FP8_PB_WO:
        wsf = ex.get_scaling_factor(wq)                                    # keeps the block amax's shape
        out.update(weight=ex.to_quantized_weight(w, wsf, fmt, block_size=wq.block_sizes[-1]), weight_scale=wsf)
    elif fmt == ex.QUANTIZATION_MXFP8 or fmt in ex._MXFP4_FORMATS:
        d = ex.export_quantized_linear(module)
        out.update(weight=d["weight"], weight_scale=d["weight_scale"])
    else:
        raise NotImplementedError(f"unified-HF export of format {fmt!r}")
    if iq.is_enabled and iq.amax is not None:
        out["input_scale"] = ex.get_activation_scaling_factor(module).squeeze()
    return out


def summarize_exclude_modules(excluded, quantized) -> list:
    """Cover the excluded module names with as few prefix wildcards as possible (``name*``, or ``name.*`` where
    ``name*`` would also match a sibling such as ``name_b``), never with one that matches a quantized module or any
    prefix of a quantized module's name.  The candidates for a name are tried from the shortest prefix, cut at dots,
    to the full name; a name already covered adds nothing."""
    blocked = set()
    for q in quantized:
        blocked.add(q)
        blocked.update(q[:i] + "*" for i in range(len(q) + 1))
    out = set()
    for name in excluded:
        options = []
        for i, c in enumerate(name):
            if c == ".":
                options += [(name[:i] + "*",), (name[:i], name[:i] + ".*")]
        options.append((name,))
        for opt in options:
            if any(w in blocked for w in opt):
                continue
            if not all(w in out for w in opt):
                out.add(opt[-1])                      # the pair (p, p.*) is written as p.* alone
            break
    return sorted(out)


def _layer_config(fmt: str, group: int) -> dict:
    algo, grouped, pqs = _ALGO.get(fmt, (fmt, False, False))
    cfg = {"quant_algo": algo}
    if grouped:
        cfg["group_size"] = group
    if pqs:
        cfg.update(has_zero_point=False, pre_quant_scale=True)
    return cfg


def get_quant_config(model: nn.Module) -> dict:
    """hf_quant_config.json (quant_utils.py:1583-1700 + process_layer_quant_config :680-789).  Modules that carry
    quantizers but stay unquantized, and embeddings (the reference attaches -- disabled -- quantizers to
    ``nn.Embedding``), are excluded.  One per-layer config gives it at the top level with the summarized
    ``exclude_modules``; more than one gives ``quant_algo: "MIXED_PRECISION"`` and the per-layer map
    ``quantized_layers``."""
    layers, excluded = {}, []
    for name, m in model.named_modules():
        if is_quantized_linear(m):
            f = ex.get_quantization_format(m)
            if f is None:
                excluded.append(name)
            else:
                bs = m.weight_quantizer.block_sizes
                layers[name] = _layer_config(f, bs.get(-1) if bs else 0)
        elif isinstance(m, nn.Embedding):
            excluded.append(name)
    q = {"quant_algo": None, "kv_cache_quant_algo": None, "quantized_layers": layers}
    distinct = {json.dumps(c, sort_keys=True) for c in layers.values()}
    if len(distinct) > 1:
        q["quant_algo"] = "MIXED_PRECISION"
    elif distinct:
        del q["quantized_layers"]
        q.update(json.loads(distinct.pop()))
        q["exclude_modules"] = summarize_exclude_modules(excluded, layers)
    return {"producer": {"name": "modelopt", "version": "b200quant"}, "quantization": q}


@torch.no_grad()
def export_hf_state_dict(model: nn.Module):
    """-> (state_dict with the unified-HF names, hf_quant_config dict).  Modifies the model's quantizer state the
    way the reference's export does (re-smoothing, unified amax)."""
    requantize_resmooth_fused_llm_layers(model)
    cfg = get_quant_config(model)
    sd = {}
    handled = set()
    for name, m in model.named_modules():
        if is_quantized_linear(m) and ex.get_quantization_format(m) is not None:
            for suffix, t in export_linear_tensors(m).items():
                sd[f"{name}.{suffix}"] = t
            pqs = getattr(m.input_quantizer, "_pre_quant_scale", None)
            if pqs is not None:
                sd[f"{name}.pre_quant_scale"] = pqs.detach()
            if m.bias is not None:
                sd[f"{name}.bias"] = m.bias.detach()
            handled.add(name)
    for key, t in model.state_dict().items():
        mod = key.rsplit(".", 1)[0]
        if mod in handled or "_quantizer" in key:
            continue
        sd[key] = t.detach()
    return sd, cfg


def export_hf_checkpoint(model: nn.Module, export_dir: str):
    """``export_hf_checkpoint`` (unified_export_hf.py:1540-1649): ``model.safetensors`` + ``hf_quant_config.json``
    (+ the HF ``config.json`` when the model has one)."""
    from safetensors.torch import save_file

    sd, cfg = export_hf_state_dict(model)
    os.makedirs(export_dir, exist_ok=True)
    save_file({k: v.contiguous().cpu() for k, v in sd.items()}, os.path.join(export_dir, "model.safetensors"),
              metadata={"format": "pt"})
    with open(os.path.join(export_dir, "hf_quant_config.json"), "w") as f:
        json.dump(cfg, f, indent=4)
    if hasattr(model, "config") and hasattr(model.config, "to_json_file"):
        model.config.to_json_file(os.path.join(export_dir, "config.json"))
    return sd, cfg


__all__ = ["export_hf_checkpoint", "export_hf_state_dict", "export_linear_tensors", "get_quant_config",
           "summarize_exclude_modules", "requantize_resmooth_fused_llm_layers", "preprocess_linear_fusion",
           "fuse_prequant_layernorm", "fuse_prequant_to_linear", "collect_shared_input_modules"]

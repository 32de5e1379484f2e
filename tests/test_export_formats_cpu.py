"""Export format labels and hf_quant_config.json for every weight format the mirror calibrates, against the reference's
export of the same tiny Llama (tests/golden/ref_export_formats*.npz, made by tools/gen_export_formats_golden.py).
Only quantizer attributes are read, so no kernel runs."""

import json

import pytest
import torch

from oracle import golden
from tools.gen_export_formats_golden import CASES, MIXED, mixed_config, tiny_llama_config


@pytest.fixture(scope="module")
def fx():
    return golden.load("ref_export_formats")


def cpu_model(fx, case):
    """The mirror's Llama on CPU with the case's quantizers configured and its pre_quant_scales in place."""
    from transformers import LlamaForCausalLM

    import model_optimizer_b200.config as cfgs
    from model_optimizer_b200.model_quant import replace_quant_module, set_quantizer_by_cfg

    model = LlamaForCausalLM(tiny_llama_config()).to(torch.bfloat16).eval()
    replace_quant_module(model)
    qcfg = mixed_config(case, cfgs.get_preset) if case in MIXED else cfgs.get_preset(case)
    set_quantizer_by_cfg(model, qcfg["quant_cfg"])
    mods = dict(model.named_modules())
    for k in fx.files:
        pre = f"{case}/in/q/"
        if k.startswith(pre) and k.endswith("._pre_quant_scale"):
            q = mods[k[len(pre):].rsplit(".", 1)[0]]
            q.pre_quant_scale = torch.from_numpy(fx[k]).to(torch.bfloat16)
    return model


@pytest.mark.parametrize("case", CASES)
def test_format_labels_match_reference(fx, case):
    from model_optimizer_b200 import export as ex

    model = cpu_model(fx, case)
    want = json.loads(str(fx[f"{case}/fmt"]))
    got = {name: ex.get_quantization_format(m) for name, m in model.named_modules() if name in want}
    assert got == want


@pytest.mark.parametrize("case", CASES)
def test_quant_config_matches_reference(fx, case):
    from model_optimizer_b200.export_hf import get_quant_config

    want = json.loads(str(fx[f"{case}/cfg"]))["quantization"]
    assert get_quant_config(cpu_model(fx, case))["quantization"] == want


def test_fixture_covers_mixed_precision_and_exclusion_summaries(fx):
    cfgs = {c: json.loads(str(fx[f"{c}/cfg"]))["quantization"] for c in CASES}
    assert all(f"{c}/error" not in fx for c in CASES)
    for c in MIXED:
        assert cfgs[c]["quant_algo"] == "MIXED_PRECISION"
        assert len({json.dumps(v, sort_keys=True) for v in cfgs[c]["quantized_layers"].values()}) == 2
    assert "model.layers.0.self_attn*" in cfgs["NVFP4_MLP_ONLY_CFG"]["exclude_modules"]
    assert "model.layers.0.self_attn.q_proj" in cfgs["NVFP4_OMLP_ONLY_CFG"]["exclude_modules"]


def test_format_label_rules():
    """The label rules around W4A8-NVFP4-FP8, and the three that changed toward the reference's: per-channel FP8,
    weight-only INT8, NVFP4 with a pre_quant_scale or a folded one."""
    from torch import nn

    import model_optimizer_b200.config as cfgs
    from model_optimizer_b200 import export as ex
    from model_optimizer_b200.model_quant import replace_quant_module, set_quantizer_by_cfg

    m = nn.Sequential(nn.Linear(64, 64))
    replace_quant_module(m)
    for preset, fmt in (("W4A8_NVFP4_FP8_CFG", "w4a8_nvfp4_fp8"), ("FP8_PER_CHANNEL_PER_TOKEN_CFG", "fp8_pc_pt"),
                        ("INT8_WEIGHT_ONLY_CFG", "int8_wo"), ("INT8_DEFAULT_CFG", "int8_sq"),
                        ("FP8_DEFAULT_CFG", "fp8"), ("NVFP4_AWQ_LITE_CFG", "nvfp4")):
        set_quantizer_by_cfg(m, cfgs.get_preset(preset)["quant_cfg"])
        assert ex.get_quantization_format(m[0]) == fmt, preset
    m[0].input_quantizer.pre_quant_scale = torch.ones(64)
    assert ex.get_quantization_format(m[0]) == "nvfp4_awq"
    delattr(m[0].input_quantizer, "_pre_quant_scale")
    m[0].fused_with_prequant = True
    assert ex.get_quantization_format(m[0]) == "nvfp4_awq"


@pytest.mark.parametrize("excluded,quantized,want", [
    (["a.b.c", "a.b.d"], ["a.e.f"], ["a.b*"]),
    (["a.b.c"], ["a.bx"], ["a.b.*"]),                         # a.b* would also match the quantized a.bx
    (["x.attn"], ["x.attn_q"], ["x.attn"]),
    (["lm_head", "model.embed_tokens"], ["model.layers.0.mlp.up_proj"], ["lm_head", "model.embed_tokens"]),
    (["m.l.0.q", "m.l.0.k", "m.l.1.q"], ["m.l.0.o", "m.l.1.o"], ["m.l.0.k", "m.l.0.q", "m.l.1.q"]),
    ([], ["a"], []),
])
def test_exclude_summary(excluded, quantized, want):
    from model_optimizer_b200.export_hf import summarize_exclude_modules

    assert summarize_exclude_modules(excluded, quantized) == want

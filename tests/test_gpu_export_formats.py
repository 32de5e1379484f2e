"""Unified-HF export of every weight format the mirror calibrates, byte for byte against the reference's
``export_hf_checkpoint`` of the same calibrated state (tests/golden/ref_export_formats*.npz, made by
tools/gen_export_formats_golden.py with the reference run on CPU): FP8 per-channel, INT8 (SmoothQuant and weight-only),
FP8 2-D blocks, MXFP8, MXFP4, W4A8-MXFP4-FP8, W4A8-NVFP4-FP8, NVFP4-AWQ, the NVFP4 MLP-only presets and two
mixed-precision models.  Each weight is packed by its kernel; the packs dequantize back to the mirror's fake quant."""

import json
import os

import numpy as np
import pytest
import torch

from oracle import golden
from tools.gen_export_formats_golden import CASES, MIXED, mixed_config, tiny_llama_config

pytestmark = pytest.mark.gpu
TD = {"torch.bfloat16": torch.bfloat16, "torch.float32": torch.float32, "torch.float16": torch.float16}
# the C-ABI entry point that packs each format's weight
PACK = {"fp8": "b200q_pack_fp8", "fp8_pc_pt": "b200q_pack_fp8", "fp8_pb_wo": "b200q_pack_fp8",
        "int8_sq": "b200q_pack_int8", "int8_wo": "b200q_pack_int8", "mxfp8": "b200q_pack_mxfp8",
        "mxfp4": "b200q_pack_mxfp4", "w4a8_mxfp4_fp8": "b200q_pack_mxfp4", "nvfp4": "b200q_pack_nvfp4",
        "nvfp4_awq": "b200q_pack_nvfp4", "w4a8_nvfp4_fp8": "b200q_pack_nvfp4_scale2"}


@pytest.fixture(scope="module")
def fx():
    return golden.load("ref_export_formats")


def build_calibrated(fx, case):
    """The mirror model in the state the reference's export started from."""
    from transformers import LlamaForCausalLM

    import model_optimizer_b200.config as cfgs
    from model_optimizer_b200.model_quant import replace_quant_module, set_quantizer_by_cfg
    from model_optimizer_b200.nn import TensorQuantizer

    model = LlamaForCausalLM(tiny_llama_config()).to(torch.bfloat16).eval()
    with torch.no_grad():
        for name, p in model.named_parameters():
            raw = fx.get(f"{case}/in/param/{name}", fx[f"base/param/{name}"])
            p.copy_(torch.from_numpy(raw.copy()).view(torch.bfloat16).reshape(p.shape))
    model = model.cuda()
    replace_quant_module(model)
    qcfg = mixed_config(case, cfgs.get_preset) if case in MIXED else cfgs.get_preset(case)
    set_quantizer_by_cfg(model, qcfg["quant_cfg"])
    mods = dict(model.named_modules())
    qdtype = json.loads(str(fx[f"{case}/in/qdtype"]))
    pre = f"{case}/in/q/"
    for k in fx.files:
        if not k.startswith(pre):
            continue
        qname, buf = k[len(pre):].rsplit(".", 1)
        q = mods.get(qname)
        if not isinstance(q, TensorQuantizer):
            continue
        t = torch.from_numpy(fx[k]).to(TD[qdtype[f"{qname}.{buf}"]]).cuda()
        if buf == "_amax":
            q.amax = t
        elif buf == "_global_amax":
            q.register_buffer("_global_amax", t)
        else:
            q._enable_pre_quant_scale = True
            q.pre_quant_scale = t
    with torch.no_grad():                                   # first forward of static-block quantizers fixes their layout
        for m in model.modules():
            wq = getattr(m, "weight_quantizer", None)
            if isinstance(wq, TensorQuantizer) and wq.is_enabled and wq.is_static_block_quant:
                wq(m.weight)
    return model


def expected(fx, case):
    meta = json.loads(str(fx[f"{case}/meta"]))
    return {k: (dt, shape, fx.get(f"{case}/out/{k}", fx.get(f"base/param/{k}"))) for k, (dt, shape) in meta.items()}


def raw_bytes(t):
    t = t.detach().contiguous().reshape(-1)
    return t.view(torch.uint8).cpu().numpy() if t.numel() else np.zeros(0, np.uint8)


def assert_state_dict_equal(sd, want):
    assert sorted(sd) == sorted(want), sorted(set(sd) ^ set(want))[:10]
    bad = []
    for k, (dt, shape, raw) in want.items():
        t = sd[k]
        assert str(t.dtype) == dt and list(t.shape) == shape, (k, t.dtype, tuple(t.shape), dt, shape)
        got = raw_bytes(t)
        if not np.array_equal(got, raw):
            bad.append((k, int((got != raw).sum()), raw.size))
    assert not bad, bad[:8]


@pytest.mark.parametrize("case", CASES)
def test_export_bytes_equal_reference(fx, case, monkeypatch):
    from model_optimizer_b200 import export as ex
    from model_optimizer_b200 import export_hf, ops

    model = build_calibrated(fx, case)
    calls = []
    real_call = ops.call
    monkeypatch.setattr(ops, "call", lambda name, *a: (calls.append(name), real_call(name, *a))[1])

    def no_torch_pack(*a, **k):
        raise AssertionError("a weight pack rounded in torch")

    monkeypatch.setattr(torch.Tensor, "round", no_torch_pack)
    monkeypatch.setattr(torch, "round", no_torch_pack)
    packs = {}
    real_linear = export_hf.export_linear_tensors

    def per_linear(m):
        calls.clear()
        out = real_linear(m)
        packs[ex.get_quantization_format(m)] = set(calls)
        return out

    monkeypatch.setattr(export_hf, "export_linear_tensors", per_linear)
    sd, cfg = export_hf.export_hf_state_dict(model)
    monkeypatch.undo()
    assert cfg["quantization"] == json.loads(str(fx[f"{case}/cfg"]))["quantization"]
    assert_state_dict_equal(sd, expected(fx, case))
    fmts = set(json.loads(str(fx[f"{case}/fmt"])).values()) - {None}
    assert set(packs) == fmts
    for fmt, names in packs.items():
        assert PACK[fmt] in names, (fmt, sorted(names))


@pytest.mark.parametrize("case", [c for c in CASES if c not in ("NVFP4_MLP_ONLY_CFG", "NVFP4_OMLP_ONLY_CFG")])
def test_from_quantized_weight_round_trip(fx, case):
    """Each exported weight dequantizes (``from_quantized_weight``, unpack kernels) to the mirror's own fake quant of
    the weight it was packed from.  Three packs round by another rule than the fake quant, so only the error size is
    checked there: the per-tensor FP8 checkpoint divides by a 0-dim scale, so the quotient is rounded to bf16 before
    the e4m3 cast (unified_export_hf.py:637-639) and about one element in sixteen lands on a tie that rounds to even;
    W4A8-NVFP4-FP8 packs against amax / 448 instead of amax / (6 * 448); the MXFP4 pack takes the E8M0 scale
    2^ceil(log2(amax / 6)) (mxfp4_tensor.py:73-75) where the MX fake quant takes 2^(floor(log2(amax)) - 2), one
    binade lower for a block maximum in (6, 8) x 2^k."""
    from model_optimizer_b200 import export as ex
    from model_optimizer_b200.export_hf import export_hf_state_dict
    from model_optimizer_b200.nn import is_quantized_linear

    model = build_calibrated(fx, case)
    sd, _ = export_hf_state_dict(model)
    seen = set()
    with torch.no_grad():
        for name, m in model.named_modules():
            if not is_quantized_linear(m) or ex.get_quantization_format(m) is None:
                continue
            fmt = ex.get_quantization_format(m)
            bs = (m.weight_quantizer.block_sizes or {}).get(-1)
            deq = ex.from_quantized_weight(sd[f"{name}.weight"], sd[f"{name}.weight_scale"], fmt, torch.bfloat16,
                                           sd.get(f"{name}.weight_scale_2"), block_size=bs).float()
            fq = m.weight_quantizer(m.weight).float()
            err = ((deq - fq).norm() / fq.norm()).item()
            if fmt in ("fp8", "w4a8_nvfp4_fp8", "mxfp4", "w4a8_mxfp4_fp8"):
                assert err < 0.2 and ((deq - m.weight.float()).norm() / m.weight.float().norm()).item() < 0.2, name
            else:
                close = torch.isclose(deq, fq, rtol=2 ** -7, atol=1e-6)
                assert close.float().mean().item() > 0.995 and err < 1e-2, (name, fmt, err)
            seen.add(fmt)
    assert seen


def test_mixed_precision_checkpoint_file_round_trip(fx, tmp_path):
    from safetensors.torch import load_file

    from model_optimizer_b200.export_hf import export_hf_checkpoint

    case = "MIXED_NVFP4_FP8PC_O_DOWN"
    sd, cfg = export_hf_checkpoint(build_calibrated(fx, case), str(tmp_path))
    assert_state_dict_equal(load_file(os.path.join(tmp_path, "model.safetensors")), expected(fx, case))
    with open(os.path.join(tmp_path, "hf_quant_config.json")) as f:
        on_disk = json.load(f)
    assert on_disk["quantization"] == json.loads(str(fx[f"{case}/cfg"]))["quantization"]
    assert on_disk["quantization"]["quant_algo"] == "MIXED_PRECISION"

"""Four-Over-Six without a GPU: the config flag and preset, the 256 / 448 normalization the quantizer hands to the
static fake quant, the compress refusal, the export scale math, and the search oracle against the reference's CPU
run (tests/golden/ref_four_over_six.npz)."""

import json
import os

import numpy as np
import pytest
import torch

from model_optimizer_b200 import config as cfgs
from model_optimizer_b200.config import QuantizerAttributeConfig
from model_optimizer_b200.nn import tensor_quantizer as tq_mod
from model_optimizer_b200.nn.tensor_quantizer import TensorQuantizer, fp8_max_for_normalization
from oracle import golden
from tools import nvfp4_mse_oracle as mo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LINEARS = ("q_proj", "k_proj", "v_proj", "o_proj")
STATIC = {"num_bits": (2, 1), "block_sizes": {-1: 16, "type": "static", "scale_bits": (4, 3)}}


def _norm(o):
    if isinstance(o, dict):
        return {str(k): _norm(v) for k, v in o.items()}
    if isinstance(o, (list, tuple)):
        return [_norm(v) for v in o]
    return o


def quantizer(four_over_six):
    bs = dict(STATIC["block_sizes"])
    if four_over_six is not None:
        bs["four_over_six"] = four_over_six
    return TensorQuantizer(QuantizerAttributeConfig(num_bits=(2, 1), block_sizes=bs))


def test_block_sizes_accepts_four_over_six_and_rejects_unknown_keys():
    c = QuantizerAttributeConfig(num_bits=(2, 1), block_sizes={-1: 16, "type": "static", "scale_bits": (4, 3),
                                                               "four_over_six": True})
    assert c.block_sizes["four_over_six"] is True
    with pytest.raises(ValueError):
        QuantizerAttributeConfig(num_bits=(2, 1), block_sizes={-1: 16, "four_over_seven": True})


def test_preset_equals_reference():
    ref = json.load(open(os.path.join(ROOT, "tests", "golden", "ref_four_over_six_preset.json")))
    assert _norm(cfgs.get_preset("NVFP4_FOUR_OVER_SIX_CFG")) == ref


@pytest.mark.parametrize("flag,want", [(None, 448.0), (False, 448.0), (True, 256.0), (1, 256.0)])
def test_fake_quant_normalization(monkeypatch, flag, want):
    """The static fake quant receives fp8_max_for_normalization (a stand-in for the kernel records it)."""
    seen = []

    def stand_in(x, amax, global_amax, quantize_block_scales, fp8_max_norm, out_dtype, pass_through_bwd):
        seen.append(fp8_max_norm)
        return x

    monkeypatch.setattr(tq_mod, "static_blockwise_fp4_fake_quant", stand_in)
    q = quantizer(flag)
    q.amax = torch.ones(4, dtype=torch.float32)
    q.register_buffer("_global_amax", torch.tensor(1.0))
    q._fake_quantize(torch.ones(4, 16))
    assert seen == [want] and fp8_max_for_normalization(q) == want


def test_compress_refuses_four_over_six():
    q = quantizer(True)
    with pytest.raises(NotImplementedError, match="Four-Over-Six"):
        q._real_quantize(torch.ones(4, 16))


@pytest.mark.parametrize("flag,norm", [(False, 448.0), (True, 256.0)])
def test_export_weight_scale_2(flag, norm):
    from model_optimizer_b200 import export

    q = quantizer(flag)
    q.amax = torch.full((4,), 3.0)
    q.register_buffer("_global_amax", torch.tensor(5.25))
    got = export.get_scaling_factor(q)
    assert torch.equal(got, torch.tensor(5.25) / (6.0 * norm))


def test_oracle_equals_fixture_four_over_six():
    g = golden.load("ref_four_over_six")
    for n in LINEARS:
        best, idx, _ = mo.search(g[f"fos/{n}/w"], g[f"fos/{n}/amax0"], g[f"fos/{n}/global_amax"],
                                 np.float32([1.0, 1.5]), 256.0, "cpu")
        assert np.array_equal(best.view(np.uint32), g[f"fos/{n}/amax"].view(np.uint32)), n
        assert np.array_equal(idx == 1, g[f"fos/{n}/chose_x1.5"]), n
        assert 0 < g[f"fos/{n}/chose_x1.5"].sum() < idx.size, n
    assert len({float(g[f"fos/{n}/global_amax"]) for n in ("q_proj", "k_proj", "v_proj")}) == 1   # shared


def test_oracle_equals_fixture_default_multipliers():
    g = golden.load("ref_four_over_six")
    best, _, _ = mo.search(g["mse39/w"], g["mse39/amax0"], g["mse39/global_amax"], g["mse39/mult"], 448.0, "cpu")
    assert np.array_equal(best.view(np.uint32), g["mse39/amax"].view(np.uint32))


def test_export_scale_2_in_fixture():
    g = golden.load("ref_four_over_six")
    for n in LINEARS:
        want = np.float32(g[f"fos/{n}/global_amax"]) / np.float32(6 * 256)
        assert g[f"fos/{n}/export/weight_scale_2"] == want, n


def test_summation_orders_differ():
    """ATen's CUDA tree (x[e] + x[e + 8], then offsets 4, 2, 1) and its CPU lane order (8 lanes of x[l] + x[l + 8]
    added to 0 in turn) round this row differently."""
    row = np.zeros((1, 16), np.float32)
    row[0, 0] = 1.0
    row[0, 8:] = 2.0 ** -24
    assert mo.block_sum(row, "cpu")[0] == np.float32(1.0)
    assert mo.block_sum(row, "cuda")[0] == np.float32(1.0 + 3 * 2.0 ** -23)


def test_c_abi_symbol():
    from model_optimizer_b200 import _lib

    assert "b200q_nvfp4_static_mse_sweep" in _lib.EXPORTED_SYMBOLS
    assert "b200q_nvfp4_static_mse_sweep(" in open(os.path.join(ROOT, "include", "b200quant.h")).read()

"""Generate tests/golden/ref_four_over_six.npz and ref_four_over_six_preset.json by running the REAL reference on CPU.

Run from the repo root where the reference tree is available:  python tools/gen_four_over_six_golden.py

Reuses the import shim of oracle/gen_golden.py.  The reference fake-quantizes static NVFP4 only through its Triton
kernel (``static_blockwise_fp4_fake_quant``); the oracle's static fake quant (``oracle_np.fake_quant_nvfp4_static``,
which the GPU tests pin to the engine's kernel and to the reference's Triton) stands in for it.  Everything around it
runs as shipped: ``mtq.quantize`` with ``NVFP4_FOUR_OVER_SIX_CFG`` (max calibration, the shared q/k/v global amax,
promotion, and ``MseCalibrator`` with its ``F.mse_loss`` / ``torch.sum`` / ``argmin``), and the ``NVFP4QTensor``
export of the calibrated weights.  The dynamic NVFP4 input quantizers need CUDA in the reference, so the model
output is taken with the input quantizers disabled (weights fake-quantized only).  Contents:

- ``preset``: NVFP4_FOUR_OVER_SIX_CFG as loaded (the JSON file);
- ``fos/*``: a q/k/v/o block in bf16 -- weights, max-calibrated and MSE-calibrated ``_amax``, ``_global_amax``,
  which blocks chose x1.5, the input and the model output, and per linear the export tensors ``weight``,
  ``weight_scale`` (E4M3 bits) and ``weight_scale_2``;
- ``mse39/*``: one static NVFP4 weight (fp8_max_for_normalization 448) through ``mse`` with the default 39
  multipliers 0.25..4.0.
"""

from __future__ import annotations

import copy
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import golden  # noqa: E402
from oracle import oracle_np as o  # noqa: E402
from oracle.gen_golden import _install_shim  # noqa: E402
from tools import nvfp4_mse_oracle as mo  # noqa: E402

LINEARS = ("q_proj", "k_proj", "v_proj", "o_proj")


def _stand_in(x, amax, global_amax=None, quantize_block_scales=True, fp8_max_for_normalization=448.0,
              out_dtype=None, *_):
    """``static_blockwise_fp4_fake_quant`` on CPU through the oracle."""
    import torch

    names = {torch.bfloat16: "bf16", torch.float16: "f16", torch.float32: "f32"}
    out_dtype = out_dtype or x.dtype
    g = None if global_amax is None else float(global_amax.float().reshape(-1)[0])
    y = o.fake_quant_nvfp4_static(x.detach().float().numpy(), amax.detach().float().numpy().reshape(-1), g,
                                  quantize_block_scales, float(fp8_max_for_normalization), names[out_dtype])
    return torch.from_numpy(y).reshape(x.shape).to(out_dtype)


def _norm(obj):
    if isinstance(obj, dict):
        return {str(k): _norm(v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return [_norm(v) for v in obj]
    return obj


def main(ref_root="/root/reference"):
    _install_shim()
    if ref_root not in sys.path:
        sys.path.insert(0, ref_root)
    import torch
    import torch.nn as nn

    import modelopt.torch.quantization as mtq
    from modelopt.torch.export import quant_utils as qu
    from modelopt.torch.quantization.nn.modules import tensor_quantizer as ref_tq

    ref_tq.static_blockwise_fp4_fake_quant = _stand_in
    out = {}

    # the oracle's CPU block-sum order is torch's on this machine
    g = torch.Generator().manual_seed(3)
    sq = (torch.randn(4096, 16, generator=g) * torch.exp(4 * torch.randn(4096, 16, generator=g))) ** 2
    assert np.array_equal(mo.block_sum(sq.numpy(), "cpu").view(np.uint32), sq.sum(dim=1).numpy().view(np.uint32))

    with open(os.path.join(golden.DIR, "ref_four_over_six_preset.json"), "w") as f:
        json.dump(_norm(mtq.NVFP4_FOUR_OVER_SIX_CFG), f, indent=1, sort_keys=True)

    class Attn(nn.Module):
        def __init__(self):
            super().__init__()
            self.q_proj, self.k_proj = nn.Linear(64, 64, bias=False), nn.Linear(64, 32, bias=False)
            self.v_proj, self.o_proj = nn.Linear(64, 32, bias=False), nn.Linear(64, 48, bias=False)

        def forward(self, x):
            return torch.cat([getattr(self, n)(x) for n in LINEARS], dim=-1)

    torch.manual_seed(0)
    model = Attn()
    with torch.no_grad():
        for i, n in enumerate(LINEARS):
            w = getattr(model, n).weight
            w.mul_(1 + 6 * (torch.rand(w.shape) < 0.03).float())          # heavy-tailed blocks
            w[0, :16] = 0                                                 # an all-zero block
            w[1, 16:32] *= 1e-6                                           # tiny blocks
            if i == 0:
                w[2, :16] = torch.tensor([4.0, 3.0, 2.0, 1.5, 1.0, 0.75, 0.5, 0.25] * 2) * w.abs().max() / 4
    model = model.to(torch.bfloat16)
    x = torch.randn(8, 64, generator=torch.Generator().manual_seed(1)).to(torch.bfloat16)
    out["fos/x"] = x.float().numpy()
    for n in LINEARS:
        out[f"fos/{n}/w"] = getattr(model, n).weight.detach().float().numpy().copy()

    cfg_max = copy.deepcopy(mtq.NVFP4_FOUR_OVER_SIX_CFG)
    cfg_max["algorithm"] = "max"
    ref_max = mtq.quantize(copy.deepcopy(model), cfg_max, None)
    mtq.quantize(model, mtq.NVFP4_FOUR_OVER_SIX_CFG, None)
    for n in LINEARS:
        wq, wq0 = getattr(model, n).weight_quantizer, getattr(ref_max, n).weight_quantizer
        a0, a1 = wq0._amax.float().reshape(-1).numpy(), wq._amax.float().reshape(-1).numpy()
        out[f"fos/{n}/amax0"], out[f"fos/{n}/amax"] = a0, a1
        out[f"fos/{n}/global_amax"] = wq.global_amax.float().reshape(()).numpy()
        out[f"fos/{n}/chose_x1.5"] = a1 != a0
        assert wq._amax.dtype == torch.float32
        best, _, _ = mo.search(out[f"fos/{n}/w"], a0, out[f"fos/{n}/global_amax"], np.float32([1.0, 1.5]), 256.0, "cpu")
        assert np.array_equal(best.view(np.uint32), a1.view(np.uint32)), n
        m = getattr(model, n)
        wsf, wsf2 = qu.get_weight_scaling_factor(m), qu.get_weight_scaling_factor_2(m)
        packed = qu.to_quantized_weight(m.weight, wsf, qu.get_quantization_format(m), wsf2, 16)
        out[f"fos/{n}/export/weight"] = packed.view(torch.uint8).numpy()
        out[f"fos/{n}/export/weight_scale"] = wsf.view(torch.uint8).numpy()
        out[f"fos/{n}/export/weight_scale_2"] = wsf2.float().reshape(()).numpy()
    for m in model.modules():
        if hasattr(m, "input_quantizer"):
            m.input_quantizer.disable()
    with torch.no_grad():
        out["fos/y"] = model(x).float().numpy()

    # ---- the default 39-multiplier search on a plain static NVFP4 weight (448) -----------------------------------
    torch.manual_seed(2)
    lin = nn.Sequential(nn.Linear(96, 40, bias=False))
    with torch.no_grad():
        lin[0].weight.mul_(1 + 10 * (torch.rand(40, 96) < 0.02).float())
    out["mse39/w"] = lin[0].weight.detach().float().numpy().copy()
    cfg = copy.deepcopy(mtq.NVFP4_W4A4_WEIGHT_MSE_FP8_SWEEP_CFG)
    cfg["algorithm"] = {"method": "mse"}
    cfg_max = copy.deepcopy(cfg)
    cfg_max["algorithm"] = "max"
    lin0 = mtq.quantize(copy.deepcopy(lin), cfg_max, None)
    mtq.quantize(lin, cfg, None)
    wq, wq0 = lin[0].weight_quantizer, lin0[0].weight_quantizer
    out["mse39/amax0"], out["mse39/amax"] = wq0._amax.float().reshape(-1).numpy(), wq._amax.float().reshape(-1).numpy()
    out["mse39/global_amax"] = wq.global_amax.float().reshape(()).numpy()
    out["mse39/mult"] = torch.linspace(0.25, 4.0, steps=39).numpy()

    golden.save("ref_four_over_six", out)
    print(f"wrote {len(out)} arrays to tests/golden/ref_four_over_six.npz and ref_four_over_six_preset.json")


if __name__ == "__main__":
    main(*sys.argv[1:])

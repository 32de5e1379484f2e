"""Generate tests/golden/ref_rotate.npz by running the REAL reference's rotation code on CPU.

Run from the repo root where the reference tree is available:  python tools/gen_rotate_golden.py [reference_root]

The reference takes the transform from the external ``fast_hadamard_transform`` package.  A stand-in module whose
``hadamard_transform(x, scale)`` is ``tools/hadamard_oracle.hadamard`` is put in ``sys.modules``; everything around
it runs as shipped: ``normalized_hadamard_transform`` (block choice, reshape, fp32 casts, error texts), the ordering
of ``rotate`` / ``rotate_back`` / disabled / ``rotate_fp32`` / ``block_size`` in ``TensorQuantizer.forward``, max
calibration and fake quant, and ``mtq.quantize`` of a 2-layer MLP.  What the fixture pins is that logic; the butterfly
order and the place of the scale inside the external package are the oracle's model of it, not verified against it.
"""

from __future__ import annotations

import copy
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import golden  # noqa: E402
from oracle.gen_golden import _install_shim  # noqa: E402
from tools.hadamard_oracle import hadamard  # noqa: E402

DTYPES = ("bf16", "f16", "f32")


def _install(ref_root):
    """The import shim of oracle/gen_golden.py plus the stand-in transform module."""
    _install_shim()
    if ref_root not in sys.path:
        sys.path.insert(0, ref_root)
    sys.modules["fast_hadamard_transform"] = stand_in_module()


def stand_in_module():
    """``fast_hadamard_transform`` with the oracle as ``hadamard_transform(x, scale)`` (x: [..., block])."""
    import torch

    names = {torch.bfloat16: "bf16", torch.float16: "f16", torch.float32: "f32"}

    def hadamard_transform(x, scale=1.0):
        y = hadamard(x.detach().float().cpu().numpy(), x.shape[-1], names[x.dtype], scale)
        return torch.from_numpy(y).to(device=x.device, dtype=x.dtype)

    m = types.ModuleType("fast_hadamard_transform")
    m.hadamard_transform = hadamard_transform
    return m


def rotated_inputs(preset):
    """A copy of a preset with ``rotate: True`` on its ``*input_quantizer`` entries."""
    cfg = copy.deepcopy(preset)
    for e in cfg["quant_cfg"]:
        if isinstance(e, dict) and e.get("quantizer_name") == "*input_quantizer" and isinstance(e.get("cfg"), dict):
            e["cfg"]["rotate"] = True
    return cfg


def main(ref_root="/root/reference"):
    _install(ref_root)
    import torch
    import torch.nn as nn

    import modelopt.torch.quantization as mtq
    from modelopt.torch.quantization.config import QuantizerAttributeConfig
    from modelopt.torch.quantization.nn import TensorQuantizer
    from modelopt.torch.quantization.nn.functional import normalized_hadamard_transform

    tdt = {"bf16": torch.bfloat16, "f16": torch.float16, "f32": torch.float32}
    out = {}
    g = torch.Generator().manual_seed(0)

    # ---- the wrapper: block choice and the fp32 cast ------------------------------------------------------------
    for name, shape, bs in (("d64", (3, 64), None), ("d96", (5, 96), None), ("d1920_b128", (2, 1920), 128),
                            ("d1536", (2, 1536), None), ("d16_b4", (7, 16), 4)):
        x = torch.randn(shape, generator=g)
        for d in DTYPES:
            xd = x.to(tdt[d])
            for fp32 in (False, True):
                y = normalized_hadamard_transform(xd, rotate_fp32=fp32, block_size=bs)
                assert y.dtype == xd.dtype
                out[f"wrap/{name}/{d}/fp32={int(fp32)}/x"] = xd.float().numpy()
                out[f"wrap/{name}/{d}/fp32={int(fp32)}/y"] = y.float().numpy()
    for name, shape, bs in (("no_pow2_divisor", (2, 7), None), ("not_pow2", (2, 96), 6),
                            ("not_divisible", (2, 96), 64)):
        try:
            normalized_hadamard_transform(torch.zeros(shape), block_size=bs)
            raise AssertionError(f"{name}: no error")
        except (RuntimeError, ValueError) as e:
            out[f"err/{name}/type"] = np.array(type(e).__name__)
            out[f"err/{name}/msg"] = np.array(str(e))

    # ---- TensorQuantizer: calibrate, then quantize, per rotation mode ---------------------------------------------
    rotations = {"rot": {"enable": True}, "back": {"enable": True, "mode": "rotate_back"},
                 "fp32b32": {"enable": True, "rotate_fp32": True, "block_size": 32}}
    formats = {"int8": {"num_bits": 8, "axis": None}, "fp8": {"num_bits": (4, 3), "axis": None},
               "int8ch": {"num_bits": 8, "axis": 0}}
    x = torch.randn(16, 128, generator=g) * (1 + 4 * (torch.rand(16, 128, generator=g) < 0.02).float())
    for d in DTYPES:
        xd = x.to(tdt[d])
        out[f"tq/{d}/x"] = xd.float().numpy()
        for fname, fcfg in formats.items():
            for rname, rot in rotations.items():
                q = TensorQuantizer(QuantizerAttributeConfig(**fcfg, rotate=rot))
                q.disable_quant()
                q.enable_calib()
                q(xd)
                q.load_calib_amax()
                q.disable_calib()
                q.enable_quant()
                key = f"tq/{d}/{fname}/{rname}"
                out[f"{key}/amax"] = q.amax.float().numpy()
                out[f"{key}/y"] = q(xd).float().numpy()
        for rname, rot in rotations.items():
            q = TensorQuantizer(QuantizerAttributeConfig(num_bits=8, rotate=rot, enable=False))
            out[f"tq/{d}/disabled/{rname}/y"] = q(xd).float().numpy()

    # ---- 2-layer MLP, INT8_DEFAULT_CFG with rotate on the input quantizers -----------------------------------------
    for d in ("f32", "bf16"):
        torch.manual_seed(1)
        model = nn.Sequential(nn.Linear(64, 128), nn.ReLU(), nn.Linear(128, 32)).to(tdt[d])
        gb = torch.Generator().manual_seed(7)
        data = [torch.randn(16, 64, generator=gb).to(tdt[d]) for _ in range(4)]
        key = f"mlp/{d}"
        for i in (0, 2):
            out[f"{key}/w{i}"] = model[i].weight.detach().float().numpy().copy()
            out[f"{key}/b{i}"] = model[i].bias.detach().float().numpy().copy()
        for i, b in enumerate(data):
            out[f"{key}/calib{i}"] = b.float().numpy()
        cfg = rotated_inputs(mtq.INT8_DEFAULT_CFG)
        mtq.quantize(model, cfg, lambda m: [m(b) for b in data])
        assert model[0].input_quantizer.rotate_is_enabled and not model[0].weight_quantizer.rotate_is_enabled
        for i in (0, 2):
            out[f"{key}/in_amax{i}"] = model[i].input_quantizer.amax.float().numpy()
            out[f"{key}/w_amax{i}"] = model[i].weight_quantizer.amax.float().numpy()
        with torch.no_grad():
            out[f"{key}/logits"] = model(data[0]).float().numpy()

    golden.save("ref_rotate", out)
    print(f"wrote {len(out)} arrays to tests/golden/ref_rotate*.npz")


if __name__ == "__main__":
    main(*sys.argv[1:])

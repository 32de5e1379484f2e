"""Generate tests/golden/ref_act_headroom.npz by running the REAL reference's ``nvfp4_act_headroom`` on CPU.

Run from the repo root where the reference tree is available:  python tools/gen_act_headroom_golden.py

Reuses the import shim of oracle/gen_golden.py.  The reference fake-quantizes dynamic NVFP4 blocks only through CUDA
code and static NVFP4 blocks only through Triton; the oracle's ``fake_quant_nvfp4`` stands in for
``tensor_quant.dynamic_block_quantize_op`` (as in tools/gen_awq_golden.py) and its ``fake_quant_nvfp4_static`` for
``static_blockwise_fp4_fake_quant`` (as in tools/gen_four_over_six_golden.py).  Everything else runs as shipped: ``mtq.quantize`` with NVFP4 inputs and weights and the
algorithm dict ``{"method": "nvfp4_act_headroom", ...}``.

The model (``Net``): ``q`` and ``k`` (40 -> 24) read the SAME tensor ``x`` whose last dim, 40, is not a multiple of 16;
``o`` (32 -> 16) reads ``relu(x[..., :32])``; ``z`` (32 -> 8) reads zeros; ``unused`` (40 -> 8) is never called.  Every
input a quantizer sees is computed exactly from the data on any device (no matmul in front of a quantizer), so the
histograms -- and therefore the amaxes -- do not depend on where the model runs.  The data spreads per-token scales
over 2^-6 .. 2^3 so that the block amaxes cover
several octaves (a range the default rho clears; a small rho does not).

Per case ``<case>/<dtype>`` (dtype f32 / bf16), arrays under that prefix:

- ``<lin>.<q>.amax`` / ``.amax_dtype`` (the ``_amax`` buffer as float32 values and the torch dtype name), absent when
  the quantizer holds none; ``<lin>.<q>.enabled``; ``<lin>.<q>.calibrator`` the calibrator's class name after the run;
- ``warnings``: the messages of the warnings that mention ``nvfp4_act_headroom``, in order;
- ``y``: the output on the held-out batch with quantization on.

``CASES`` maps each case to its algorithm options and whether its weights are static NVFP4 (the weight-scale searches
``mse`` with ``fp8_scale_sweep`` and ``local_hessian`` refine static NVFP4 weights).  Weights, biases and data are stored
once per dtype under ``model/<dtype>/``.
"""

from __future__ import annotations

import copy
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import golden  # noqa: E402
from oracle import oracle_np as o  # noqa: E402
from oracle.gen_golden import _install_shim  # noqa: E402

LINEARS = ("q", "k", "o", "z", "unused")
QUANTIZERS = ("input_quantizer", "weight_quantizer")
DTYPES = ("f32", "bf16")
CASES = {
    "default": ({}, False),
    "upper100": ({"anchor_percentile": 5.0, "upper_percentile": 100.0}, False),
    "small_rho": ({"rho": 2.0}, False),
    "w_max": ({"weight_scale_algorithm": {"method": "max"}}, True),
    "w_mse": ({"weight_scale_algorithm": {"method": "mse", "fp8_scale_sweep": True}}, True),
    "w_local_hessian": ({"weight_scale_algorithm": {"method": "local_hessian"}}, True),
}
_NVFP4_DYN = {"num_bits": (2, 1), "block_sizes": {-1: 16, "type": "dynamic", "scale_bits": (4, 3)}}
_NVFP4_STATIC = {"num_bits": (2, 1), "block_sizes": {-1: 16, "type": "static", "scale_bits": (4, 3)}}


def quant_cfg(static_weights: bool, algorithm: dict) -> dict:
    """The config both the reference and the mirror run: NVFP4 dynamic inputs, NVFP4 weights."""
    return {"quant_cfg": [{"quantizer_name": "*", "enable": False},
                          {"quantizer_name": "*input_quantizer", "cfg": copy.deepcopy(_NVFP4_DYN)},
                          {"quantizer_name": "*weight_quantizer",
                           "cfg": copy.deepcopy(_NVFP4_STATIC if static_weights else _NVFP4_DYN)}],
            "algorithm": {"method": "nvfp4_act_headroom", **copy.deepcopy(algorithm)}}


def net(dtype):
    """The model, built identically by the reference run and the tests."""
    import torch
    import torch.nn as nn

    class Net(nn.Module):
        def __init__(self):
            super().__init__()
            self.q, self.k = nn.Linear(40, 24), nn.Linear(40, 24)
            self.o, self.z, self.unused = nn.Linear(32, 16), nn.Linear(32, 8), nn.Linear(40, 8)

        def forward(self, x):
            h = torch.relu(x[..., :32])
            return torch.cat([self.q(x) + self.k(x), self.o(h), self.z(torch.zeros_like(h))], -1)

    torch.manual_seed(21)
    return Net().to(dtype)


def data(dtype):
    import torch

    g = torch.Generator().manual_seed(22)

    def batch(b, t):
        scale = torch.exp2(torch.randint(-6, 4, (b, t, 1), generator=g).float())
        return (torch.randn(b, t, 40, generator=g) * scale).to(dtype)

    return [batch(2, 24) for _ in range(3)], batch(1, 8)


def _stand_in(inputs, block_size, amax, num_bits, exponent_bits, scale_num_bits, scale_exponent_bits):
    """``dynamic_block_quantize_op`` for NVFP4 (E2M1 elements, E4M3 block scales, blocks of 16) on CPU."""
    import torch

    assert (num_bits, exponent_bits, scale_num_bits, scale_exponent_bits, block_size) == (4, 2, 8, 4, 16)
    names = {torch.bfloat16: "bf16", torch.float16: "f16", torch.float32: "f32"}
    x = inputs.detach().float().numpy()
    g = np.float32(np.abs(x).max()) if amax is None else np.float32(amax.detach().float().reshape(-1)[0])
    y = o.fake_quant_nvfp4(x, g, names[inputs.dtype])
    return torch.from_numpy(y).reshape(inputs.shape).to(inputs.dtype)


def _f32(t):
    return t.detach().float().cpu().numpy().copy()


def main(ref_root="/root/reference"):
    _install_shim()
    if ref_root not in sys.path:
        sys.path.insert(0, ref_root)
    import torch

    import modelopt.torch.quantization as mtq
    from modelopt.torch.quantization import tensor_quant as ref_tensor_quant
    from modelopt.torch.quantization.nn.modules import tensor_quantizer as ref_tq

    from tools.gen_four_over_six_golden import _stand_in as _static_stand_in

    ref_tensor_quant.dynamic_block_quantize_op = _stand_in
    ref_tq.static_blockwise_fp4_fake_quant = _static_stand_in
    torch.set_num_threads(1)                                 # one summation order on every CPU
    tdt = {"f32": torch.float32, "bf16": torch.bfloat16}
    out = {}
    for d in DTYPES:
        base = net(tdt[d])
        calib, test = data(tdt[d])
        for n in LINEARS:
            out[f"model/{d}/{n}.weight"] = _f32(getattr(base, n).weight)
            out[f"model/{d}/{n}.bias"] = _f32(getattr(base, n).bias)
        out[f"model/{d}/calib"] = np.stack([_f32(x) for x in calib])
        out[f"model/{d}/test"] = _f32(test)
        for case, (algo, static_w) in CASES.items():
            key = f"{case}/{d}"
            model = copy.deepcopy(base)
            with warnings.catch_warnings(record=True) as caught:
                warnings.simplefilter("always")
                mtq.quantize(model, quant_cfg(static_w, algo), lambda m: [m(x) for x in calib])
            msgs = [str(w.message) for w in caught if "nvfp4_act_headroom" in str(w.message)]
            out[f"{key}/warnings"] = np.array(msgs, dtype=np.str_)
            for n in LINEARS:
                lin = getattr(model, n)
                for qn in QUANTIZERS:
                    q = getattr(lin, qn)
                    p = f"{key}/{n}.{qn}"
                    out[p + ".enabled"] = np.array(q.is_enabled)
                    out[p + ".calibrator"] = np.array(type(q._calibrator).__name__)
                    a = getattr(q, "_amax", None)
                    if isinstance(a, torch.Tensor):
                        out[p + ".amax"] = _f32(a)
                        out[p + ".amax_dtype"] = np.array(str(a.dtype))
            with torch.no_grad():
                out[f"{key}/y"] = _f32(model(test))
            print(key, {n: out.get(f"{key}/{n}.input_quantizer.amax") for n in LINEARS}, len(msgs), "warnings")
    golden.save("ref_act_headroom", out)
    print(f"wrote {len(out)} arrays to tests/golden/ref_act_headroom.npz")


if __name__ == "__main__":
    main(*sys.argv[1:])

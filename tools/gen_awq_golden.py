"""Generate tests/golden/ref_awq.npz by running the REAL reference's ``awq_clip`` / ``awq_lite`` on CPU.

Run from the repo root where the reference tree is available:  python tools/gen_awq_golden.py

Reuses the import shim of oracle/gen_golden.py.  The reference fake-quantizes dynamic NVFP4 blocks only through
CUDA code (its Triton kernel or the MX extension); the oracle's ``fake_quant_nvfp4`` (pinned to the engine's kernel
and to the reference's Triton kernel by the GPU tests) stands in for ``tensor_quant.dynamic_block_quantize_op``.
Everything else runs as shipped: ``mtq.quantize`` with the preset, the algorithm dict carrying ``debug=True`` and
small ``max_co_batch_size`` / ``max_tokens_per_batch`` so that the co-batch loop and the strided token subsample run.

The model (``Net``): ``l0`` 128 -> 136 (cin a multiple of 128 and of 16; co 136 > max_co_batch_size 32, ragged last
co batch), ReLU, ``l1`` 136 -> 64 (ragged cin: padded for blocks of 16 and of 128), and ``l2`` 136 -> 16, which the
forward never calls.  Weights carry a few x8 outlier input columns, activations a few x6 channels, so that clipping
and smoothing pay off.  Calibration data: three [2, 20, 128] batches (40 rows > max_tokens_per_batch 16, stride 2);
the held-out batch is [1, 8, 128].

Per case ``<preset>/<dtype>`` (dtype f32 / bf16), arrays under that prefix:

- ``<lin>.<q>.amax`` / ``.amax_dtype`` (the ``_amax`` buffer, float32 values and the torch dtype name), absent when the
  quantizer holds none; ``<lin>.<q>.enabled``; ``<lin>.<q>.pqs`` the ``_pre_quant_scale`` when there is one;
- ``<lin>.weight_after`` the weight after smoothing (awq_lite; awq_clip leaves every weight as it was);
- awq_clip: ``<lin>.clip.loss`` [n_ratio, *amax shape] (the debug ``awq_clip.loss``), ``clip.ratios``,
  ``<lin>.clip.w_amax``, ``<lin>.clip.num_tokens``, ``<lin>.clip.best`` (absent when postprocessing was skipped);
- awq_lite: ``<lin>.lite.loss`` [n_alpha], ``lite.alphas``, ``<lin>.lite.best_alpha`` (NaN when not searched),
  ``<lin>.lite.act_scale``, ``<lin>.lite.weight_scale``, ``<lin>.lite.enabled``;
- ``y`` the output on the held-out batch with quantization on.

The model weights, biases and the data are stored once per dtype under ``model/<dtype>/``.
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

LINEARS = ("l0", "l1", "l2")
QUANTIZERS = ("input_quantizer", "weight_quantizer", "output_quantizer")
CLIP_PRESETS = ("INT4_BLOCKWISE_WEIGHT_ONLY_CFG", "NVFP4_AWQ_CLIP_CFG", "INT8_DEFAULT_CFG", "FP8_DEFAULT_CFG")
LITE_PRESETS = ("INT4_AWQ_CFG", "NVFP4_AWQ_LITE_CFG")
CLIP_ARGS = {"max_co_batch_size": 32, "max_tokens_per_batch": 16, "debug": True}
LITE_ARGS = {"alpha_step": 0.1, "debug": True}
DTYPES = ("f32", "bf16")


def net(dtype):
    """The 3-linear model, built identically by the reference run and the GPU test."""
    import torch
    import torch.nn as nn

    class Net(nn.Module):
        def __init__(self):
            super().__init__()
            self.l0, self.l1, self.l2 = nn.Linear(128, 136), nn.Linear(136, 64), nn.Linear(136, 16)

        def forward(self, x):
            return self.l1(torch.relu(self.l0(x)))           # l2 is never called

    torch.manual_seed(11)
    m = Net()
    with torch.no_grad():
        m.l0.weight[:, 3::41] *= 8                           # outlier input columns
        m.l1.weight[:, 7::37] *= 8
        m.l2.weight[:, 5::41] *= 8
    return m.to(dtype)


def data(dtype):
    import torch

    g = torch.Generator().manual_seed(12)
    col = torch.ones(128)
    col[::29] = 6.0                                          # salient activation channels
    calib = [(torch.randn(2, 20, 128, generator=g) * col).to(dtype) for _ in range(3)]
    test = (torch.randn(1, 8, 128, generator=g) * col).to(dtype)
    return calib, test


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

    ref_tensor_quant.dynamic_block_quantize_op = _stand_in
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

        for preset in CLIP_PRESETS + LITE_PRESETS:
            key = f"{preset}/{d}"
            cfg = copy.deepcopy(getattr(mtq, preset))
            if preset in CLIP_PRESETS:
                cfg["algorithm"] = {"method": "awq_clip", **CLIP_ARGS}
            else:
                cfg["algorithm"] = {"method": "awq_lite", **LITE_ARGS}
            model = copy.deepcopy(base)
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                mtq.quantize(model, cfg, lambda m: [m(x) for x in calib])
            for n in LINEARS:
                lin = getattr(model, n)
                for qn in QUANTIZERS:
                    q = getattr(lin, qn)
                    p = f"{key}/{n}.{qn}"
                    out[p + ".enabled"] = np.array(q.is_enabled)
                    a = getattr(q, "_amax", None)
                    if isinstance(a, torch.Tensor):
                        out[p + ".amax"] = _f32(a)
                        out[p + ".amax_dtype"] = np.array(str(a.dtype))
                    s = getattr(q, "_pre_quant_scale", None)
                    if isinstance(s, torch.Tensor):
                        out[p + ".pqs"] = _f32(s)
                        out[p + ".pqs_dtype"] = np.array(str(s.dtype))
                if preset in LITE_PRESETS:
                    out[f"{key}/{n}.weight_after"] = _f32(lin.weight)
                else:
                    assert torch.equal(lin.weight, getattr(base, n).weight), (key, n)
                st = getattr(lin, "awq_clip", None)
                if st is not None:
                    ratios = list(st.loss)
                    out[f"{key}/clip.ratios"] = np.array(ratios, dtype=np.float64)
                    out[f"{key}/{n}.clip.loss"] = np.stack([_f32(st.loss[r]) for r in ratios])
                    out[f"{key}/{n}.clip.w_amax"] = _f32(st.w_amax)
                    out[f"{key}/{n}.clip.num_tokens"] = np.array(st.num_tokens)
                    if st.best_clip_val is not None:
                        out[f"{key}/{n}.clip.best"] = _f32(st.best_clip_val)
                st = getattr(lin, "awq_lite", None)
                if st is not None:
                    alphas = list(st.loss)
                    out[f"{key}/lite.alphas"] = np.array(alphas, dtype=np.float64)
                    out[f"{key}/{n}.lite.loss"] = np.array([float(st.loss[a]) for a in alphas], dtype=np.float64)
                    out[f"{key}/{n}.lite.best_alpha"] = np.float64(np.nan if st.best_alpha is None else st.best_alpha)
                    out[f"{key}/{n}.lite.enabled"] = np.array(st.is_enabled)
                    if isinstance(st.act_scale, torch.Tensor):
                        out[f"{key}/{n}.lite.act_scale"] = _f32(st.act_scale)
                    out[f"{key}/{n}.lite.weight_scale"] = _f32(st.weight_scale)
            with torch.no_grad():
                out[f"{key}/y"] = _f32(model(test))
            print(key, "y[0,0,:3]", out[f"{key}/y"][0, 0, :3])
    golden.save("ref_awq", out)
    print(f"wrote {len(out)} arrays to tests/golden/ref_awq.npz")


if __name__ == "__main__":
    main(*sys.argv[1:])

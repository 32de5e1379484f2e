"""Generate tests/golden/ref_hessian_sweep.npz by running the REAL reference on CPU.

Run from the repo root where the reference tree is available:  python tools/gen_hessian_sweep_golden.py

Reuses the import shim of oracle/gen_golden.py.  Contents:

- ``hess/<cin>/*`` (a): ``_LocalHessianAccumulator.accumulate`` over three batches (3-D, 2-D, 3-D activations) for
  cin in {16, 48, 256}; the activations ``x<i>`` and ``normalized_hessian()`` as uint32 bits.  At cin 48 the second
  cin block's activations are all zero.
- ``sweep/<dtype>/<cout>x<cin>/*`` (b): ``NVFP4MSECalibrator(..., error_func=acc.build_error_func(), hessian=H)``
  on CPU, which runs the reference's 126-step sweep with the einsum metric, with a torch static NVFP4 fake quant as
  ``quant_func`` (the ``qf`` of gen_golden.main_algos: block scale ``amax / 6``, no FP8 rounding).  Weights ``w``
  (Gaussian with heavy-tailed blocks, exact E2M1 ties at power-of-two candidate scales, an all-zero block, a -0.0
  block; global amax exactly 1), the global amax ``g``, the candidates ``cand`` (e4m3 / 448), the winners ``best``
  and the per-candidate losses ``losses`` ([126, blocks] of the first ``loss_rows`` rows).
- ``mult/<cfg>/<dtype>/*`` (c): ``mtq.quantize`` with ``{"method": "local_hessian", "fp8_scale_sweep": False}`` on
  the config-1 MLP (64 -> 128 -> 32, oracle/gen_golden.py) with INT8 per-channel (INT8_DEFAULT_CFG) and FP8
  per-tensor (FP8_DEFAULT_CFG) weights, fp32 and bf16: the weights, the calibration data, per linear the weight
  quantizer's ``_amax`` after max calibration (``amax_max``) and after the search (``amax``), and its normalized
  Hessian (``hess``).
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
from oracle.gen_golden import _install_shim  # noqa: E402

CINS = (16, 48, 256)
SWEEP_CASES = [(d, cout, cin) for d in ("bf16", "f32") for cout in (5, 300) for cin in CINS
               if not (cout == 300 and cin == 256)]
LOSS_ROWS = 20


def activations(cin):
    import torch

    g = torch.Generator().manual_seed(100 + cin)
    col = 1 + 3 * torch.rand(cin, generator=g)                   # a different Hessian per cin block
    xs = [torch.randn(2, 6, cin, generator=g) * col, torch.randn(10, cin, generator=g) * col,
          torch.randn(1, 7, cin, generator=g) * col]
    if cin == 48:
        for x in xs:
            x[..., 16:32] = 0                                    # a cin block with all-zero activations
    return xs


def weight(cout, cin, dtype, seed):
    import torch

    g = torch.Generator().manual_seed(seed)
    w = torch.randn(cout, cin, generator=g)
    w = w * (1 + 20 * (torch.rand(cout, cin, generator=g) < 0.01).float())     # heavy tail
    w = w / w.abs().max()
    w[0, 0] = 1.0                                                # global amax exactly 1: candidate scales c / 6
    ties = torch.tensor([0.25, 0.75, 1.25, 1.75, 2.5, 3.5, 5.0, 0.5] * 2)
    ties[1::2] *= -1
    for r in range(1, cout, 7):                                   # exact E2M1 ties at s = 2^-3 (c = 0.75), 2^-4 ...
        w[r, (r % (cin // 16)) * 16:][:16] = ties * 2.0 ** -(3 + r % 3)
    w[min(2, cout - 1), :16] = 0.0                               # an all-zero block
    w[min(3, cout - 1), -16:] = -0.0                             # a -0.0 block
    w[min(4, cout - 1), -16::3] = -0.0
    return w.to(dtype)


def main(ref_root="/root/reference"):
    _install_shim()
    if ref_root not in sys.path:
        sys.path.insert(0, ref_root)
    warnings.filterwarnings("ignore")
    import torch
    import torch.nn as nn

    import modelopt.torch.quantization as mtq
    from modelopt.torch.quantization.calib.mse import MseCalibrator, NVFP4MSECalibrator
    from modelopt.torch.quantization.model_calib import _LocalHessianAccumulator
    from modelopt.torch.quantization.utils import reduce_amax, reduce_block_amax

    torch.manual_seed(0)
    out = {}
    dtypes = {"bf16": torch.bfloat16, "f32": torch.float32}

    # ---- (a) the accumulator ---------------------------------------------------------------------------------------
    for cin in CINS:
        acc = _LocalHessianAccumulator(8, cin, 16)
        for i, x in enumerate(activations(cin)):
            acc.accumulate(x)
            out[f"hess/{cin}/x{i}"] = x.numpy().copy()
        out[f"hess/{cin}/h_bits"] = acc.normalized_hessian().numpy().view(np.uint32).copy()

    # ---- (b) the reference Hessian sweep ---------------------------------------------------------------------------
    def qf(t, a):  # static NVFP4 fake quant in pure torch (oracle/gen_golden.py main_algos)
        scale = (a.float() / 6.0)
        s = torch.where(scale == 0, torch.ones_like(scale), scale)
        absx = t.abs() / s
        b = torch.tensor([0.25, 0.75, 1.25, 1.75, 2.5, 3.5, 5.0])
        vals = torch.tensor([0, 0.5, 1, 1.5, 2, 3, 4, 6.0])
        idx = torch.bucketize(absx, b, right=False)
        tie_up = (absx == 0.75) | (absx == 1.75) | (absx == 3.5)
        return torch.sign(t) * vals[idx + tie_up.long()] * s

    for i, (d, cout, cin) in enumerate(SWEEP_CASES):
        w = weight(cout, cin, dtypes[d], 1000 + i)
        acc = _LocalHessianAccumulator(cout, cin, 16)
        for x in activations(cin):
            acc.accumulate(x)
        hess = acc.normalized_hessian()
        assert np.array_equal(hess.numpy().view(np.uint32), out[f"hess/{cin}/h_bits"])
        ef = acc.build_error_func(keep_buffer=True)
        bam = reduce_block_amax(w, {-1: 16}).float().reshape(-1, 1)
        g = reduce_amax(w).float()
        assert float(g) == 1.0
        xb = w.reshape(-1, 16)
        cal = NVFP4MSECalibrator(amax=bam, global_amax=g, axis=0, quant_func=qf, error_func=ef, hessian=hess)
        cal.collect(xb)                                          # CPU: the reference 126-step sweep
        best = cal.compute_amax().float().reshape(-1)
        # the same sweep step by step, to keep the per-candidate losses that collect() releases
        twin = NVFP4MSECalibrator(amax=bam, global_amax=g, axis=0, quant_func=qf, error_func=ef, hessian=hess)
        MseCalibrator.collect(twin, xb)
        losses = torch.stack(twin._losses_sum)
        assert torch.equal(MseCalibrator.compute_amax(twin).float().reshape(-1), best)
        key = f"sweep/{d}/{cout}x{cin}"
        out[f"{key}/w"] = w.float().numpy()
        out[f"{key}/g"] = g.numpy()
        out[f"{key}/cand"] = twin._candidates.numpy().copy()
        out[f"{key}/best"] = best.numpy()
        rows = min(cout, LOSS_ROWS)
        out[f"{key}/losses"] = losses[:, : rows * (cin // 16)].numpy().copy()
        out[f"{key}/loss_rows"] = np.int64(rows)

    # ---- (c) the multiplier search under the Hessian metric ------------------------------------------------------
    for cname in ("INT8_DEFAULT_CFG", "FP8_DEFAULT_CFG"):
        for d, dtype in dtypes.items():
            torch.manual_seed(1)
            model = nn.Sequential(nn.Linear(64, 128), nn.ReLU(), nn.Linear(128, 32)).to(dtype)
            gen = torch.Generator().manual_seed(7)
            data = [torch.randn(16, 64, generator=gen).to(dtype) for _ in range(4)]
            key = f"mult/{cname}/{d}"
            out[f"{key}/data"] = torch.stack(data).float().numpy()

            def loop(m):
                for x in data:
                    m(x)

            for li in (0, 2):
                out[f"{key}/l{li}/w"] = model[li].weight.detach().float().numpy().copy()
                out[f"{key}/l{li}/b"] = model[li].bias.detach().float().numpy().copy()
            cfg_max = copy.deepcopy(getattr(mtq, cname))
            cfg_max["algorithm"] = "max"
            ref_max = mtq.quantize(copy.deepcopy(model), cfg_max, loop)
            cfg = copy.deepcopy(getattr(mtq, cname))
            cfg["algorithm"] = {"method": "local_hessian", "fp8_scale_sweep": False, "debug": True}
            mtq.quantize(model, cfg, loop)
            accs = model._local_hessian_accumulators
            for li in (0, 2):
                q, q0 = model[li].weight_quantizer, ref_max[li].weight_quantizer
                out[f"{key}/l{li}/amax_max"] = q0._amax.detach().float().numpy().copy()
                out[f"{key}/l{li}/amax"] = q._amax.detach().float().numpy().copy()
                out[f"{key}/l{li}/hess"] = accs[id(q)].normalized_hessian().numpy().copy()
                assert str(q._amax.dtype) == str(q0._amax.dtype)
            moved = float(np.mean(out[f"{key}/l0/amax"] != out[f"{key}/l0/amax_max"]))
            print(f"{key}: amax moved off max calibration: {moved:.2f} (l0)")

    golden.save("ref_hessian_sweep", out)
    total = sum(os.path.getsize(os.path.join(golden.DIR, f)) for f in os.listdir(golden.DIR)
                if f.startswith("ref_hessian_sweep"))
    print(f"wrote {len(out)} arrays to tests/golden/ref_hessian_sweep*.npz ({total} bytes)")


if __name__ == "__main__":
    main(*sys.argv[1:])

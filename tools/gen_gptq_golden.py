"""Generate tests/golden/ref_gptq.npz by running the REAL reference's GPTQ code on CPU.

Run from the repo root where the reference tree is available:  python tools/gen_gptq_golden.py

Reuses the import shim of oracle/gen_golden.py.  What runs as shipped (modelopt/torch/quantization/utils/calib_utils.py):
``update_hessian`` over several batches (and with zero tokens), ``compute_hessian_inverse`` with a dead weight column
and on a Hessian that is not positive definite, and ``gptq_blockwise_update`` over one block (block_size =
in_features in {16, 64, 128}: no trailing GEMM), for fp32 and bf16 source weights.  The quantizer is the reference's
``TensorQuantizer`` max-calibrated on the source weight: INT8 per row, FP8 per tensor (on CPU the reference takes its
eager FP8 rule, ``fl(1 / amax) * 448``) and INT4 with static 128-element blocks.  On CPU, ATen's ``addr_`` rounds like
one fused multiply-add.

The reference cannot fake-quantize NVFP4 on CPU (dynamic blocks need CUDA, static blocks Triton).  For the two NVFP4
formats the oracle's full-matrix NVFP4 fake quant (tools/gptq_oracle.py) stands in as ``quantize_fn``: those runs pin
the reference's GPTQ loop around the quantizer (the working copy, which column is kept, the error scaling and the
rank-1 update), not the NVFP4 rounding itself, which the GPU tests pin against the engine's kernels.
"""

from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import golden  # noqa: E402
from oracle.gen_golden import _install_shim  # noqa: E402
from tools import gptq_oracle as orc  # noqa: E402


def main():
    _install_shim()
    import torch

    from modelopt.torch.quantization.config import QuantizerAttributeConfig
    from modelopt.torch.quantization.nn import TensorQuantizer
    from modelopt.torch.quantization.utils import calib_utils as cu

    out = {}
    g = torch.Generator().manual_seed(0)

    # ---- update_hessian: three batches, one batch, zero tokens --------------------------------------------------
    xs = [torch.randn(2, 7, 32, generator=g) for _ in range(3)]
    h, n = torch.zeros(32, 32), 0
    for i, x in enumerate(xs):
        out[f"hess/x{i}"] = x.numpy()
        h, n = cu.update_hessian(x, h, n)
    out["hess/h3"], out["hess/n3"] = h.numpy().copy(), np.array(n)
    h1, n1 = cu.update_hessian(torch.cat([x.reshape(-1, 32) for x in xs]), torch.zeros(32, 32), 0)
    out["hess/h1"], out["hess/n1"] = h1.numpy(), np.array(n1)

    # ---- compute_hessian_inverse: dead column, and the identity fallback ------------------------------------------
    x = torch.randn(256, 32, generator=g)
    hh, _ = cu.update_hessian(x, torch.zeros(32, 32), 0)
    w = torch.randn(16, 32, generator=g)
    w[:, 5] = 0
    out["hinv/h"], out["hinv/w"] = hh.numpy(), w.numpy()
    out["hinv/u"] = cu.compute_hessian_inverse(hh, w, 0.01).contiguous().numpy()
    out["hinv/u_bad"] = cu.compute_hessian_inverse(-torch.eye(8), torch.ones(4, 8), 0.01).contiguous().numpy()

    # ---- one GPTQ block ---------------------------------------------------------------------------------------------
    formats = {"int8_row": {"num_bits": 8, "axis": 0}, "fp8": {"num_bits": (4, 3), "axis": None},
               "int4_b128": {"num_bits": 4, "block_sizes": {-1: 128, "type": "static"}}}
    for nb in (16, 64, 128):
        x = torch.randn(4 * nb, nb, generator=g)
        hb, _ = cu.update_hessian(x, torch.zeros(nb, nb), 0)
        for sdt in ("f32", "bf16"):
            w_src = torch.randn(24, nb, generator=g) * 0.05
            w_src[3] = 0                                         # a zero row
            if sdt == "bf16":
                w_src = w_src.to(torch.bfloat16)
            weight = w_src.float().clone()
            u = cu.compute_hessian_inverse(hb, weight, 0.01)
            key = f"block/{nb}/{sdt}"
            out[f"{key}/w"] = weight.numpy().copy()
            out[f"{key}/u"] = u.contiguous().numpy()
            for fname, fcfg in formats.items():
                if fname == "int4_b128" and nb % 128:
                    continue
                q = TensorQuantizer(QuantizerAttributeConfig(**fcfg))
                q.disable_quant()
                q.enable_calib()
                q(w_src)
                q.load_calib_amax()
                q.disable_calib()
                q.enable_quant()
                wk = weight.clone()
                cu.gptq_blockwise_update(wk, u, nb, q)
                out[f"{key}/{fname}/amax"] = q.amax.float().numpy()
                out[f"{key}/{fname}/out"] = wk.numpy()
            # NVFP4: the oracle's fake quant stands in for the quantizer
            blocks = weight.reshape(-1, 16).abs().amax(dim=1)
            gamax = float(blocks.max())
            for fname, fmt, amax in (("nvfp4_static", orc.FMT_NVFP4_STATIC, blocks.numpy()),
                                     ("nvfp4_dynamic", orc.FMT_NVFP4_DYNAMIC, np.array([gamax], np.float32))):
                def quantize_fn(m, fmt=fmt, amax=amax):
                    return torch.from_numpy(orc.fake_quant_nvfp4(m.numpy(), fmt, amax, gamax))

                wk = weight.clone()
                cu.gptq_blockwise_update(wk, u, nb, quantize_fn)
                out[f"{key}/{fname}/amax"] = np.asarray(amax, np.float32)
                out[f"{key}/{fname}/global_amax"] = np.array(gamax, np.float32)
                out[f"{key}/{fname}/out"] = wk.numpy()

    golden.save("ref_gptq", out)
    print(f"wrote {len(out)} arrays to tests/golden/ref_gptq.npz")


if __name__ == "__main__":
    main()

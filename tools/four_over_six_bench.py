"""Static NVFP4 multiplier-search timings on Llama-3-8B weight shapes (bf16): the fused search
(``b200q_nvfp4_static_mse_sweep``, one launch per weight) against the composed path the reference's ``MseCalibrator``
runs on the GPU (per candidate: an fp32 copy, the static fake quant, ``F.mse_loss``, ``sum(dim=1)``; then
``argmin`` and the product), for the Four-Over-Six pair {1.0, 1.5} at 256 and the default 39 multipliers at 448, and
the whole-model ``mse_calibrate`` of ``NVFP4_FOUR_OVER_SIX_CFG`` over one Llama-3-8B decoder layer's linears.
Checks that the fused and the composed search give bit-identical amaxes.

    python tools/four_over_six_bench.py [--shapes 4096x4096,1024x4096,...] [--iters 20] [--out FILE]

Kernel times are CUDA events over ``--iters`` launches after a warm-up.  GB/s counts the weight read once (2 bytes
per element) plus the fp32 amax read and write (8 bytes per 16-element block) over the kernel time.  Prints one JSON
object (with the card name and its power limit) and writes it to --out when given."""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from model_optimizer_b200 import model_quant, ops  # noqa: E402
from model_optimizer_b200.config import get_preset  # noqa: E402

HBM_GBS = 3350.0     # H100 SXM data sheet, HBM3


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def events_ms(fn, iters):
    fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def composed(w, a0, g, mult, norm):
    """MseCalibrator.collect + compute_amax (calib/mse.py:84-172) as torch runs it on the GPU."""
    losses = []
    for m in mult:
        x = w.reshape(-1, 16).to(torch.float32)
        xq = ops.fake_quant_nvfp4_static(x, a0 * m, g, True, norm)
        losses.append(F.mse_loss(x, xq, reduction="none").sum(dim=1))
    return a0 * mult[torch.argmin(torch.stack(losses), dim=0)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="4096x4096,1024x4096,14336x4096,4096x14336")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("four_over_six_bench needs a CUDA device")
    torch.cuda.set_device(0)
    res = {"device": torch.cuda.get_device_name(0), "power_limit": power_limit(), "results": [], "model": None}
    for shape in a.shapes.split(","):
        out_f, in_f = (int(v) for v in shape.split("x"))
        g = torch.Generator(device="cuda").manual_seed(out_f + in_f)
        w = (torch.randn(out_f, in_f, device="cuda", generator=g) * 0.02).to(torch.bfloat16)
        a0 = w.reshape(-1, 16).abs().amax(dim=1).float()
        gam = a0.max().reshape(1)
        n_blocks = a0.numel()
        for name, mult, norm in (("four_over_six", torch.linspace(1.0, 1.5, 2, device="cuda"), 256.0),
                                 ("default_39", torch.linspace(0.25, 4.0, 39, device="cuda"), 448.0)):
            fused_ms = events_ms(lambda: ops.nvfp4_static_mse_sweep(w, a0, gam, mult, norm), a.iters)
            comp_ms = events_ms(lambda: composed(w, a0, gam, mult, norm), max(2, a.iters // 10))
            got, want = ops.nvfp4_static_mse_sweep(w, a0, gam, mult, norm), composed(w, a0, gam, mult, norm)
            gb = (w.numel() * 2 + n_blocks * 8) / 1e9
            row = {"shape": [out_f, in_f], "search": name, "candidates": mult.numel(), "fp8_max_norm": norm,
                   "fused_ms": round(fused_ms, 4), "composed_ms": round(comp_ms, 3),
                   "speedup": round(comp_ms / fused_ms, 1), "fused_GBps": round(gb / (fused_ms / 1e3), 1),
                   "fused_share_of_hbm": round(gb / (fused_ms / 1e3) / HBM_GBS, 3),
                   "fused_elements_per_s": float(f"{w.numel() / (fused_ms / 1e3):.4g}"),
                   "bit_identical": bool(torch.equal(got.view(torch.int32), want.view(torch.int32)))}
            res["results"].append(row)
            print(json.dumps(row), flush=True)
        del w, a0
        torch.cuda.empty_cache()

    # whole-model mse_calibrate of the 4/6 preset: one Llama-3-8B decoder layer's linears (q/k/v share a global amax)
    layer = torch.nn.ModuleDict({"q_proj": torch.nn.Linear(4096, 4096, bias=False),
                                 "k_proj": torch.nn.Linear(4096, 1024, bias=False),
                                 "v_proj": torch.nn.Linear(4096, 1024, bias=False),
                                 "o_proj": torch.nn.Linear(4096, 4096, bias=False),
                                 "gate_proj": torch.nn.Linear(4096, 14336, bias=False),
                                 "up_proj": torch.nn.Linear(4096, 14336, bias=False),
                                 "down_proj": torch.nn.Linear(14336, 4096, bias=False)}).to("cuda", torch.bfloat16)
    model_quant.quantize(layer, get_preset("NVFP4_FOUR_OVER_SIX_CFG"), None)          # warm-up
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    model_quant.calibrate(layer, get_preset("NVFP4_FOUR_OVER_SIX_CFG")["algorithm"], None)
    e.record()
    torch.cuda.synchronize()
    n_x15 = sum(int((m.weight_quantizer._amax != m.weight.reshape(-1, 16).abs().amax(dim=1).float().reshape(
        m.weight_quantizer._amax.shape)).sum()) for m in layer.values())
    n_all = sum(m.weight.numel() // 16 for m in layer.values())
    res["model"] = {"what": "mse_calibrate(NVFP4_FOUR_OVER_SIX_CFG), one Llama-3-8B decoder layer (7 linears)",
                    "ms": round(s.elapsed_time(e), 3), "blocks": n_all, "blocks_x1.5": n_x15}
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

"""GPTQ weight-update timings on Llama-3-8B weight shapes: the kernel path (one b200q_gptq_block launch per 128-column
block plus the trailing cuBLAS addmm_) against the composed loop (a full-matrix fake quant per column, as the
reference's unfused gptq_blockwise_update runs it), with the split of the kernel path into in-block kernel, trailing
addmm_ and the Cholesky steps of compute_hessian_inverse.  Checks that both paths give bit-identical weights.

    python tools/gptq_bench.py [--shapes 4096x4096,1024x4096,...] [--formats nvfp4_static,int4_b128] [--out FILE]

Prints one JSON object (with the card name and its power limit) and writes it to --out when given."""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from model_optimizer_b200 import model_calib, ops  # noqa: E402
from model_optimizer_b200.config import QuantizerAttributeConfig  # noqa: E402
from model_optimizer_b200.nn import TensorQuantizer  # noqa: E402

FORMATS = {"nvfp4_static": {"num_bits": (2, 1), "block_sizes": {-1: 16, "type": "static", "scale_bits": (4, 3)}},
           "int4_b128": {"num_bits": 4, "block_sizes": {-1: 128, "type": "static"}}}


def quantizer(fmt, w):
    q = TensorQuantizer(QuantizerAttributeConfig(**FORMATS[fmt])).cuda()
    q.disable_quant()
    q.enable_calib()
    q(w)
    q.load_calib_amax()
    q.disable_calib()
    q.enable_quant()
    blocks = q._amax.float()                  # promoted static blocks keep fp32 amax
    delattr(q, "_amax")
    q.amax = blocks
    if q.is_nvfp4_static:
        g = torch.zeros(1, dtype=torch.float32, device=w.device)
        ops.amax_per_tensor_(g, q._amax.contiguous())
        q.register_buffer("_global_amax", g.reshape(()))
    return q


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def kernel_path(weight, h_inv, block_size, q, desc):
    """ops.gptq_blockwise_update with CUDA events around every launch: (in-block ms, addmm ms)."""
    evs = []
    n = weight.shape[1]
    for bs in range(0, n, block_size):
        be = min(bs + block_size, n)
        e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        e0.record()
        errs = ops.gptq_block_update(weight[:, bs:be], h_inv[bs:be, bs:be], col0=bs, **desc)
        e1.record()
        weight[:, be:].addmm_(errs, h_inv[bs:be, be:], alpha=-1)
        e2.record()
        evs.append((e0, e1, e2))
    torch.cuda.synchronize()
    return sum(a.elapsed_time(b) for a, b, _ in evs), sum(b.elapsed_time(c) for _, b, c in evs)


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="4096x4096,1024x4096,14336x4096,4096x14336")
    ap.add_argument("--formats", default="nvfp4_static,int4_b128")
    ap.add_argument("--block-size", type=int, default=128)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-composed", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    res = {"device": torch.cuda.get_device_name(0), "power_limit": power_limit(), "block_size": a.block_size,
           "results": []}
    for shape in a.shapes.split(","):
        out_f, in_f = (int(v) for v in shape.split("x"))
        g = torch.Generator(device="cuda").manual_seed(out_f + in_f)
        w0 = (torch.randn(out_f, in_f, device="cuda", generator=g) * 0.02).to(torch.bfloat16)
        x = torch.randn(2048, in_f, device="cuda", generator=g)
        h, _ = model_calib.update_hessian(x, torch.zeros(in_f, in_f, device="cuda"), 0)
        del x
        for fmt in a.formats.split(","):
            q = quantizer(fmt, w0)
            weight = w0.float()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            h_inv = model_calib.compute_hessian_inverse(h, weight, 0.01)   # two Cholesky steps + cholesky_inverse
            torch.cuda.synchronize()
            chol_ms = (time.perf_counter() - t0) * 1e3
            desc = ops.gptq_quantizer_desc(q, weight.shape, a.block_size, weight.device)
            kernel_path(weight.clone(), h_inv, a.block_size, q, desc)              # warm-up
            best = None
            for _ in range(a.reps):
                wk = weight.clone()
                total = timed(lambda: ops.gptq_blockwise_update(wk, h_inv, a.block_size, q, desc=desc))
                best = total if best is None else min(best, total)
            wk2 = weight.clone()
            inblock, addmm = kernel_path(wk2, h_inv, a.block_size, q, desc)
            row = {"shape": [out_f, in_f], "format": fmt, "kernel_path_ms": round(best, 3),
                   "in_block_kernel_ms": round(inblock, 3), "trailing_addmm_ms": round(addmm, 3),
                   "hessian_inverse_ms": round(chol_ms, 3)}
            if not a.no_composed:
                wc = weight.clone()
                row["composed_ms"] = round(timed(lambda: model_calib.gptq_blockwise_update_composed(
                    wc, h_inv, a.block_size, q)), 1)
                row["speedup"] = round(row["composed_ms"] / best, 1)
                row["bit_identical"] = bool(torch.equal(wc.view(torch.int32), wk.view(torch.int32)))
            res["results"].append(row)
            print(json.dumps(row), flush=True)
            del q, h_inv
        torch.cuda.empty_cache()
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

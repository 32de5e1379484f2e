"""Input-rotation kernels on the card this runs on: the Hadamard transform against torch ``copy_`` (the read + write
ceiling of the same bytes), and the fused rotate + NVFP4 fake quant (with and without rotate_back) against the
composed transform -> fake quant (-> transform) sequence.

Times each case with CUDA events over a window of warmed back-to-back launches (at least --reps, and enough for
--window-ms of GPU time), --rounds rounds with the variants interleaved, and reports the median round.  Rates count
4 B per bf16 element (one read, one write) for every variant, so the composed sequence's extra passes show as a lower
rate.  Also checks that the fused and composed outputs are bit-identical at
the timed sizes.  Prints one JSON line with the card's name, power limit and maximum SM clock, read in the same run.

usage: python tools/rotate_bench.py [--reps 50] [--window-ms 200] [--rounds 5]"""

from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.fq_ceiling import card  # noqa: E402

SHAPES = [("act_16384x4096_B4096", (16384, 4096), 4096), ("act_16384x4096_B128", (16384, 4096), 128),
          ("kv_8x8x4096x128_B128", (8, 8, 4096, 128), 128), ("moe_16384x1536_auto", (16384, 1536), None)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--window-ms", type=float, default=200.0, help="least GPU time per timed window")
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()

    import torch

    from model_optimizer_b200 import ops
    from model_optimizer_b200.nn.functional import rotate_block_size

    if not torch.cuda.is_available():
        raise SystemExit("rotate_bench.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)

    def window(fn, reps):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(reps):
            fn()
        end.record()
        end.synchronize()
        return start.elapsed_time(end) / reps * 1e-3

    def launches(fn):
        """Launches per window: at least --reps and enough for --window-ms, from a warmed probe of 10."""
        for _ in range(3):
            fn()
        return max(args.reps, int(args.window_ms * 1e-3 / window(fn, 10)) + 1)

    results = {}
    for name, shape, block in SHAPES:
        g = torch.Generator(device=dev).manual_seed(0)
        x = torch.randn(shape, device=dev, generator=g).to(torch.bfloat16)
        bs = rotate_block_size(shape[-1], block)
        y = torch.empty_like(x)
        amax = torch.zeros(1, dtype=torch.float32, device=dev)
        ops.hadamard(x, bs, amax)
        amax = amax.to(torch.bfloat16)
        variants = {
            "copy": lambda: y.copy_(x),
            "hadamard": lambda: ops.hadamard(x, bs),
            "fused_nvfp4": lambda: ops.fake_quant_nvfp4_rotated(x, bs, amax, False),
            "composed_nvfp4": lambda: ops.fake_quant_nvfp4(ops.hadamard(x, bs), amax),
            "fused_nvfp4_back": lambda: ops.fake_quant_nvfp4_rotated(x, bs, amax, True),
            "composed_nvfp4_back": lambda: ops.hadamard(ops.fake_quant_nvfp4(ops.hadamard(x, bs), amax), bs),
        }
        same = all(torch.equal(variants[f"fused_nvfp4{s}"]().view(torch.int16),
                               variants[f"composed_nvfp4{s}"]().view(torch.int16)) for s in ("", "_back"))
        reps = {k: launches(fn) for k, fn in variants.items()}
        rounds = {k: [] for k in variants}
        for _ in range(args.rounds):
            for k, fn in variants.items():
                rounds[k].append(window(fn, reps[k]))
        nbytes = 4 * x.numel()
        r = {"block": bs, "fused_equals_composed": same}
        for k, ts in rounds.items():
            t = statistics.median(ts)
            r[k] = {"us": round(t * 1e6, 2), "GBps_at_4B": round(nbytes / t / 1e9, 1), "launches": reps[k],
                    "spread_us": [round(min(ts) * 1e6, 2), round(max(ts) * 1e6, 2)]}
        r["hadamard_vs_copy"] = round(statistics.median(rounds["copy"]) / statistics.median(rounds["hadamard"]), 3)
        for s in ("", "_back"):
            r[f"fused_speedup{s}"] = round(statistics.median(rounds[f"composed_nvfp4{s}"]) /
                                           statistics.median(rounds[f"fused_nvfp4{s}"]), 3)
        results[name] = r
        del x, y
        torch.cuda.empty_cache()
    print(json.dumps({"card": card(dev), "window_ms": args.window_ms, "min_reps": args.reps, "rounds": args.rounds,
                      "results": results}))


if __name__ == "__main__":
    main()

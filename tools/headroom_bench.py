"""NVFP4 activation-headroom collect timings for the Llama-3-8B plan on one GPU (bf16 activations, 224 input
quantizers): the 224 per-quantizer ``b200q_nvfp4_block_log2_hist`` launches (the engine's ``grouped=False`` collect),
the one grouped ``b200q_nvfp4_block_log2_hist_multi`` launch (``grouped=True``), and, as a bandwidth reference, the
grouped max collect ``amax_per_tensor_multi_`` over the same tensors.  Checks that the grouped and per-quantizer
launches give identical histograms and running maxima.

    python tools/headroom_bench.py [--tokens 4096] [--rounds 7] [--reps 5] [--out FILE]

Each variant is one CUDA graph; the rounds alternate the three, each round times ``--reps`` replays with CUDA events.
Reports per variant the median and the min / max over rounds of the per-step time, and GB/s counting 2 bytes per
activation element read once, against the H100 SXM data sheet's 3.35 TB/s.  Also the host time of the engine's
``finish`` (one device-to-host copy of the histogram table and 224 percentile evaluations).  Prints one JSON object
with the card name and its power limit and writes it to --out when given."""

from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from model_optimizer_b200 import ops  # noqa: E402
from model_optimizer_b200.engine import LLAMA3_8B, ShardedPTQEngine  # noqa: E402
from tools.four_over_six_bench import HBM_GBS, power_limit  # noqa: E402


def capture(fn, side):
    fn()                                        # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
        fn()
    return g


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=4096)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("headroom_bench needs a GPU")
    torch.cuda.set_device(0)
    eng = ShardedPTQEngine(LLAMA3_8B, args.tokens, calib="nvfp4_act_headroom", grouped=True)
    acts = eng.alloc_activations(seed=0)
    n = len(eng.quantizers)
    elems = sum(x.numel() for x in acts)
    nbytes = elems * acts[0].element_size()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    slots = torch.zeros(n, dtype=torch.float32, device="cuda")
    amax_table = ops.TensorTable(acts, list(range(n)), unit="vec32")

    def per_quantizer():
        for (_, q, _), x in zip(eng.quantizers, acts):
            q._calibrator.collect(x)

    variants = {"per_quantizer_hist": per_quantizer,
                "grouped_hist": lambda: eng.collect(acts),
                "grouped_amax": lambda: ops.amax_per_tensor_multi_(slots, amax_table)}
    # the two histogram paths must agree exactly (one step each from zero)
    res_check = {}
    for k in ("per_quantizer_hist", "grouped_hist"):
        eng.reset()
        variants[k]()
        torch.cuda.synchronize()
        res_check[k] = (eng.hist.clone(), eng.running_max.clone())
    same = torch.equal(*[v[0] for v in res_check.values()]) and torch.equal(*[v[1] for v in res_check.values()])
    graphs = {k: capture(fn, side) for k, fn in variants.items()}
    times = {k: [] for k in graphs}
    for _ in range(args.rounds):
        for k, g in graphs.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            g.replay()
            s.record()
            for _ in range(args.reps):
                g.replay()
            e.record()
            torch.cuda.synchronize()
            times[k].append(s.elapsed_time(e) / args.reps)
    eng.reset()
    eng.collect(acts)
    torch.cuda.synchronize()
    fin = []
    for _ in range(5):
        t0 = time.perf_counter()
        eng.finish()
        fin.append((time.perf_counter() - t0) * 1e3)
    out = {"device": torch.cuda.get_device_name(0), "power_limit": power_limit(), "plan": LLAMA3_8B.name,
           "tokens": args.tokens, "quantizers": n, "act_bytes_per_step": nbytes, "identical_hist": same,
           "rounds": args.rounds, "reps": args.reps, "hbm_datasheet_gbs": HBM_GBS, "variants": {},
           "finish_host_ms": {"median": statistics.median(fin), "min": min(fin), "max": max(fin)}}
    for k, ts in times.items():
        med = statistics.median(ts)
        out["variants"][k] = {"median_ms": med, "min_ms": min(ts), "max_ms": max(ts),
                              "gbs": nbytes / med / 1e6, "share_of_datasheet": nbytes / med / 1e6 / HBM_GBS}
    s = json.dumps(out, indent=1)
    print(s)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s)
    if not same:
        raise SystemExit("grouped and per-quantizer histograms differ")


if __name__ == "__main__":
    main()

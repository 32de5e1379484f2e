"""How close the grouped NVFP4 fake quant of bench.py's step comes to the read + write bandwidth this card reaches on
the same access pattern.

Builds the bench's one-GPU workload exactly (ShardedPTQEngine over Llama-3-8B: 224 bf16 activations [4096, cin], the
ring of 4 output buffers, one grouped launch per phase) and times, with CUDA events over CUDA-graph replays:
  (a) the grouped NVFP4 fake quant, which is also the calibration collect (reads 2 B, writes 2 B per element);
  (b) torch copy_ over the same source / destination pairs, one launch per pair: the read + write ceiling of this
      access pattern on this card;
  (c) the fix-up after it in the steady state: no exported amax changes, so it only rewrites the output-ring ranges
      that earlier entries of the grid also write (ops.live_block_ranges).
The three are interleaved over --rounds rounds of --reps replays each (after a warm-up); the median round is reported.
Prints one JSON line with GB/s, each phase's fraction of (b), and the card's name, power limit and maximum SM clock
read in the same run.

usage: python tools/fq_ceiling.py [--reps 20] [--rounds 3]"""

from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card(dev):
    import torch

    try:
        uuid = f"GPU-{torch.cuda.get_device_properties(dev).uuid}"
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", uuid], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = (s.strip() for s in q.split(","))
        return {"name": name, "power_limit": power, "sm_clock_max": clock}
    except Exception as e:  # noqa: BLE001
        return {"error": repr(e)[:200]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20, help="graph replays per timed round (at least 20)")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if args.reps < 20 or args.rounds < 1:
        ap.error("--reps must be at least 20 and --rounds at least 1")

    import torch

    from model_optimizer_b200.engine import LLAMA3_8B, ShardedPTQEngine

    if not torch.cuda.is_available():
        raise SystemExit("fq_ceiling.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    tokens = 4096
    eng = ShardedPTQEngine(LLAMA3_8B, tokens, "nvfp4", torch.bfloat16, dev)
    acts = eng.alloc_activations(seed=0)
    outs = eng.alloc_outputs(4)
    g = eng.capture(acts, outs)
    # one full step, so that the fake quant runs with the calibrated amax of every quantizer, as in the bench
    eng.step_graph()

    n = len(outs)
    pairs = [(x, outs[i % n][: x.numel()].view_as(x)) for i, x in enumerate(acts)]
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        for x, y in pairs:
            y.copy_(x)
    torch.cuda.synchronize(dev)
    g_copy = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g_copy, stream=side):
        for x, y in pairs:
            y.copy_(x)

    b_fixup, b_fq = eng.act_bytes_per_step()
    cases = {"fake_quant": (g["fake_quant"], b_fq), "copy": (g_copy, b_fq), "fixup": (g["collect"], b_fixup)}
    for gr, _ in cases.values():
        for _ in range(3):
            gr.replay()
    torch.cuda.synchronize(dev)
    ms = {k: [] for k in cases}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for k, (gr, _) in cases.items():
            e0.record()
            for _ in range(args.reps):
                gr.replay()
            e1.record()
            torch.cuda.synchronize(dev)
            ms[k].append(e0.elapsed_time(e1) / args.reps)
    res = {}
    for k, (_, nbytes) in cases.items():
        m = statistics.median(ms[k])
        res[k] = {"ms": round(m, 4), "bytes": nbytes, "ms_rounds": [round(v, 4) for v in ms[k]]}
        if nbytes:
            res[k]["GBps"] = round(nbytes / (m * 1e-3) / 1e9, 1)
    res["fake_quant"]["frac_of_copy"] = round(res["fake_quant"]["GBps"] / res["copy"]["GBps"], 4)
    print(json.dumps({"tool": "fq_ceiling", "card": card(dev),"tensors": len(acts), "tokens": tokens,
                      "reps": args.reps, "rounds": args.rounds, **res,
                      "what": "grouped NVFP4 fake quant + collect (a), torch copy_ over the same src/dst pairs (b) and "
                              "the steady-state fix-up (c) of bench.py's Llama-3-8B step, CUDA-graph replays timed with "
                              "CUDA events; frac_of_copy = GB/s over (b)'s GB/s"}), flush=True)


if __name__ == "__main__":
    main()

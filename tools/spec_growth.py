"""What the speculative collect + fake quant step costs when amaxes grow, against the three-phase grouped step it
replaced.

Builds bench.py's one-GPU workload (ShardedPTQEngine over Llama-3-8B: 224 bf16 activations [4096, cin], a ring of 4
output buffers) twice over the same activations:
  new: the engine's graphs -- fused collect + fake quant (speculative amax) -> fix-up -> export;
  old: collect (ops.amax_per_tensor_multi_) -> export -> fake quant (ops.fake_quant_nvfp4_multi), captured here into
       CUDA graphs over the same activations with their own arena, amax arena and output ring.
For each growth schedule (0 %, ~7 % and 100 % of the tensors set a new running max every step) both arms start from
reset and run the same steps, alternating old / new step by step.  Growth is forced between steps, outside the timed
event pair, by writing 2 x (current running max) into the first element of each chosen tensor.  Reports the median ms
per step of each arm, the fix-up's redo count, whether both arms left identical fp32 arenas, amax arenas and output
buffers (bit for bit), and the card's name, power limit and maximum SM clock read in the same run.

usage: python tools/spec_growth.py [--steps 12] [--warmup 3]"""

from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=12, help="timed steps per arm and schedule")
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import torch

    from model_optimizer_b200 import ops
    from model_optimizer_b200.engine import LLAMA3_8B, ShardedPTQEngine, _lib_call_export
    from tools.fq_ceiling import card

    if not torch.cuda.is_available():
        raise SystemExit("spec_growth.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    eng = ShardedPTQEngine(LLAMA3_8B, 4096, "nvfp4", torch.bfloat16, dev)
    acts = eng.alloc_activations(seed=0)
    outs = eng.alloc_outputs(4)
    g_new = eng.capture(acts, outs)

    # the old three-phase grouped step over the same activations, with state of its own
    idx = {n: i for i, n in enumerate(eng.arena.names())}
    slots = [idx[qn] for qn, _, _ in eng.quantizers]
    arena_old = torch.zeros_like(eng.arena.freeze())
    amax_old = torch.zeros_like(eng.amax_arena)
    outs_old = eng.alloc_outputs(4)
    ys_old = [outs_old[i % 4][: x.numel()].view_as(x) for i, x in enumerate(acts)]
    t_collect = ops.TensorTable(acts, slots, None, "vec32")
    t_fq = ops.TensorTable(acts, slots, ys_old, "block16")
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    phases = (lambda: ops.amax_per_tensor_multi_(arena_old, t_collect),
              lambda: _lib_call_export(arena_old, amax_old),
              lambda: ops.fake_quant_nvfp4_multi(t_fq, amax_old))
    with torch.cuda.stream(side):
        for f in phases:
            f()
    torch.cuda.synchronize(dev)
    g_old = []
    for f in phases:
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=side):
            f()
        g_old.append(gr)

    def step_old():
        for gr in g_old:
            gr.replay()

    def step_new():
        eng.step_graph()

    def grow(chosen):
        arena = eng.arena.freeze()
        for i in chosen:
            acts[i].view(-1)[:1].copy_(arena[slots[i]:slots[i] + 1] * 2)

    def reset():
        eng.reset()
        arena_old.zero_()
        amax_old.zero_()
        for o in outs + outs_old:
            o.zero_()

    n = len(acts)
    schedules = {"0%": [], "7%": list(range(0, n, 14)), "100%": list(range(n))}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(fn):
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize(dev)
        return e0.elapsed_time(e1)

    res = {}
    for name, chosen in schedules.items():
        reset()
        ms = {"old": [], "new": []}
        for s in range(args.warmup + args.steps):
            if s > 0:
                grow(chosen)      # the first step grows every amax anyway (from reset)
            torch.cuda.synchronize(dev)
            t_old, t_new = timed(step_old), timed(step_new)
            if s >= args.warmup:
                ms["old"].append(t_old)
                ms["new"].append(t_new)
        torch.cuda.synchronize(dev)
        same = (torch.equal(eng.arena.freeze().view(torch.int32), arena_old.view(torch.int32))
                and torch.equal(eng.amax_arena.view(torch.int16), amax_old.view(torch.int16))
                and all(torch.equal(a.view(torch.int16), b.view(torch.int16)) for a, b in zip(outs, outs_old)))
        m_old, m_new = statistics.median(ms["old"]), statistics.median(ms["new"])
        res[name] = {"tensors_growing_per_step": len(chosen), "old_ms": round(m_old, 4), "new_ms": round(m_new, 4),
                     "new_over_old": round(m_new / m_old, 4), "redo_count": int(eng.redo_count),
                     "identical": bool(same),
                     "old_ms_steps": [round(v, 4) for v in ms["old"]], "new_ms_steps": [round(v, 4) for v in ms["new"]]}
    print(json.dumps({"tool": "spec_growth", "card": card(dev), "tensors": n, "tokens": 4096, "steps": args.steps,
                      "warmup": args.warmup, **res,
                      "what": "ms per step (CUDA events, median over steps) of the old collect -> export -> fake quant "
                              "grouped step and the new fused collect + fake quant -> fix-up -> export step on bench.py's "
                              "Llama-3-8B buffers, alternated step by step; redo_count = quantizers redone by the fix-up "
                              "over warm-up + timed steps; identical = arenas, amax arenas and all output buffers of the "
                              "two arms equal bit for bit at the end"}), flush=True)


if __name__ == "__main__":
    main()

"""The grouped engine step -- fused collect + fake quant with the previous step's amax, exact fix-up, export -- against
the per-quantizer collect -> export -> fake quant step, bit for bit after every step of a sequence that exercises the
speculation: from reset, the same batch again, a lower batch, growth in some / all tensors, inf and NaN, all-zero
tensors.  Compared: the fp32 arena, the exported amax arena and the FULL content of every output buffer; the fix-up's
redo counter must count exactly the quantizers whose exported amax changed."""

import pytest
import torch

from model_optimizer_b200 import ops
from model_optimizer_b200.engine import TINY, ModelPlan, ShardedPTQEngine

pytestmark = pytest.mark.gpu

LLAMA_2L = ModelPlan("llama-3-8b-2-layers", 4096, 14336, 2, 1024)   # Llama-3-8B shapes, 14 quantizers


def _bits(t):
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()])


def _engines(plan, tokens, dtype, n_ring):
    fused = ShardedPTQEngine(plan, tokens, "nvfp4", dtype, "cuda", grouped=True)
    ref = ShardedPTQEngine(plan, tokens, "nvfp4", dtype, "cuda", grouped=False)
    acts = fused.alloc_activations(seed=11)
    n = n_ring or len(fused.quantizers)
    res = []
    for eng in (fused, ref):
        outs = eng.alloc_outputs(n)
        for o in outs:
            o.zero_()                    # the tails of the ring are never written: start both sides equal
        eng.capture(acts, outs)          # both engines read the SAME activation buffers
        res.append(outs)
    return fused, ref, acts, res[0], res[1]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32], ids=["bf16", "f16", "f32"])
@pytest.mark.parametrize("n_ring", [4, None], ids=["ring4", "one_per_quantizer"])
@pytest.mark.parametrize("plan,tokens", [(TINY, 256), (LLAMA_2L, 64)], ids=["tiny", "llama8b_2layers"])
def test_fused_step_equals_sequential_step(plan, tokens, dtype, n_ring):
    fused, ref, acts, outs_f, outs_r = _engines(plan, tokens, dtype, n_ring)
    n = len(acts)
    idx = {name: i for i, name in enumerate(fused.arena.names())}
    slots = torch.tensor([idx[qn] for qn, _, _ in fused.quantizers], device="cuda")

    def step(what, expect_redo=None):
        before = _bits(ref.amax_arena[slots]).clone()
        r0 = int(fused.redo_count)
        fused.step_graph()
        ref.step_graph()
        torch.cuda.synchronize()
        changed = int((_bits(ref.amax_arena[slots]) != before).sum())
        assert torch.equal(_bits(fused.arena.freeze()), _bits(ref.arena.freeze())), what
        assert torch.equal(_bits(fused.amax_arena), _bits(ref.amax_arena)), what
        for k, (a, b) in enumerate(zip(outs_f, outs_r)):
            assert torch.equal(_bits(a), _bits(b)), f"{what}: output buffer {k}"
        assert int(fused.redo_count) - r0 == changed, what
        if expect_redo is not None:
            assert changed == expect_redo, what

    step("from reset", expect_redo=n)
    step("same batch again", expect_redo=0)
    for x in acts:
        x.mul_(0.5)
    step("lower batch", expect_redo=0)
    subset = list(range(1, n, 3))
    for i in subset:
        x = acts[i].view(-1)
        x[7] = x.abs().max().float() * 4
    step("growth in a subset", expect_redo=len(subset))
    for x in acts:
        x.mul_(3)
    step("growth in all tensors", expect_redo=n)
    acts[2].view(-1)[5] = float("inf")
    acts[4].view(-1)[9] = float("inf")
    acts[4].view(-1)[100] = float("nan")
    step("inf and NaN", expect_redo=2)
    step("inf and NaN again", expect_redo=0)
    acts[0].zero_()
    step("an all-zero tensor", expect_redo=0)
    for eng in (fused, ref):
        eng.reset()
    acts[1].zero_()
    step("all-zero tensors from reset", expect_redo=n - 2)


def test_capture_refuses_outputs_that_overlap_inputs():
    eng = ShardedPTQEngine(TINY, 64, "nvfp4", torch.bfloat16, "cuda", grouped=True)
    acts = eng.alloc_activations(seed=1)
    outs = [acts[-1].view(-1)] + eng.alloc_outputs(3)     # entry 0 would write over the last entry's input
    with pytest.raises(ops.B200QuantError, match="overlaps an input"):
        eng.capture(acts, outs)

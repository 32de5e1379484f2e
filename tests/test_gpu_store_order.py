"""Store order of the fused collect + fake quant into output buffers that several entries share: the tiles an entry
writes last run in a second launch, pre-flagged tiles are rewritten by the fix-up.  Every case compares, bit for bit, the full output
buffers (and for the engine the fp32 arena and the exported amax) with the sequential collect -> export -> fake quant."""

import pytest
import torch

from model_optimizer_b200 import ops
from model_optimizer_b200.engine import TINY, ShardedPTQEngine

pytestmark = pytest.mark.gpu


def _bits(t):
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()])


def _sequence(plan, tokens, dtype, n_ring):
    fused = ShardedPTQEngine(plan, tokens, "nvfp4", dtype, "cuda", grouped=True)
    ref = ShardedPTQEngine(plan, tokens, "nvfp4", dtype, "cuda", grouped=False)
    acts = fused.alloc_activations(seed=23)
    outs_f, outs_r = fused.alloc_outputs(n_ring), ref.alloc_outputs(n_ring)
    for o in outs_f + outs_r:
        o.zero_()
    fused.capture(acts, outs_f)
    ref.capture(acts, outs_r)
    (table,) = fused._graphs["tables"]

    def step(what):
        fused.step_graph()
        ref.step_graph()
        torch.cuda.synchronize()
        assert torch.equal(_bits(fused.arena.freeze()), _bits(ref.arena.freeze())), what
        assert torch.equal(_bits(fused.amax_arena), _bits(ref.amax_arena)), what
        for k, (a, b) in enumerate(zip(outs_f, outs_r)):
            assert torch.equal(_bits(a), _bits(b)), f"{what}: output buffer {k}"

    step("from reset")
    step("same batch again")
    for i in range(1, len(acts), 3):
        x = acts[i].view(-1)
        x[7] = x.abs().max().float() * 4
    step("growth in a subset")
    for x in acts:
        x.mul_(0.5)
    step("lower batch")
    acts[2].view(-1)[5] = float("inf")
    acts[3].view(-1)[100] = float("nan")
    step("inf and NaN")
    acts[0].zero_()
    step("an all-zero tensor")
    return table


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32], ids=["bf16", "f16", "f32"])
@pytest.mark.parametrize("tokens,n_ring", [(40, 4), (40, 3), (256, 4)], ids=["40tok_ring4", "40tok_ring3", "256tok_ring4"])
def test_engine_steps_equal_sequential(tokens, n_ring, dtype):
    # TINY at 40 tokens: entries of 640 and 1280 blocks, live bounds at block 640, inside tile 1 (pre-flagged tiles)
    table = _sequence(TINY, tokens, dtype, n_ring)
    assert len(table.passes) == 2
    if tokens == 40:
        assert table.n_pieces > 0 and table.fixup_bytes > 0
    else:
        assert table.n_pieces == 0 and table.fixup_bytes == 0


def _sequential(xs, buf, amax):
    """The shared buffer as per-tensor fake quant launches in table order leave it."""
    want = torch.zeros_like(buf)
    for i, x in enumerate(xs):
        want[: x.numel()] = ops.fake_quant_nvfp4(x, amax[i:i + 1]).view(-1)
    return want


@pytest.mark.parametrize("shape_sets", [
    [(16, 256)],                                     # a single entry
    [(64, 512), (64, 256), (32, 512), (48, 128)],    # a few tiles in one shared buffer: far fewer than the grid's CTAs
    [(40, 256), (40, 512), (40, 256)],               # live bounds inside tiles
], ids=["single_entry", "few_tiles", "unaligned"])
def test_small_tables(shape_sets):
    g = torch.Generator(device="cuda").manual_seed(3)
    xs = [torch.randn(s, device="cuda", generator=g).to(torch.bfloat16) for s in shape_sets]
    buf = torch.zeros(max(x.numel() for x in xs), dtype=torch.bfloat16, device="cuda")
    ys = [buf[: x.numel()].view_as(x) for x in xs]
    table = ops.TensorTable(xs, None, ys, "block16", fused=True)
    slots = torch.zeros(len(xs), dtype=torch.float32, device="cuda")
    amax = torch.zeros_like(slots)
    redo = torch.zeros(1, dtype=torch.int32, device="cuda")
    for rnd in range(3):
        if rnd == 2:
            xs[-1].mul_(3)                               # the last entry's amax grows: it is redone
        ops.collect_fake_quant_nvfp4_multi(table, slots, amax)
        ops.fake_quant_nvfp4_multi_fixup(table, slots, amax, redo)
        amax.copy_(slots)
        torch.cuda.synchronize()
        assert torch.equal(slots, torch.stack([x.abs().max().float() for x in xs]))
        assert torch.equal(_bits(buf), _bits(_sequential(xs, buf, amax))), f"round {rnd}"
    assert int(redo) == len(xs) + 1

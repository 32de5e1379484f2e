"""The grouped NVFP4 fake quant maps each whole 512-block tile of a 16-bit tensor lane-contiguously, two lanes per
16-element block (nvfp4.cu dyn_fq_tile), and the partial last tile of an entry one thread per block.  Blocks whose
halves differ where the block max and the quantizer branch -- NaN in one half, an all-NaN half or block, inf next to
NaN, -0.0, block scales outside the exact-division window -- must come out of both grouped launches (plain and
collect) bit for bit as the single-tensor kernel, which keeps one thread per block, writes them; the collect must
leave the slots the amax kernel leaves."""

import pytest
import torch

from model_optimizer_b200 import ops

pytestmark = pytest.mark.gpu

NAN, INF = float("nan"), float("inf")


def _bits(t):
    return t.view({2: torch.int16, 4: torch.int32}[t.element_size()])


def _special_blocks(n_blocks, seed):
    """[n_blocks, 16] fp32 normals with every 5th block rewritten by one of the cases below, in turn"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n_blocks, 16, generator=g) * 3.0
    cases = [
        lambda b: b.__setitem__(3, NAN),                        # NaN in the low half
        lambda b: b.__setitem__(12, NAN),                       # NaN in the high half
        lambda b: b[:8].fill_(NAN),                             # all-NaN low half, finite high half
        lambda b: b[8:].fill_(NAN),                             # all-NaN high half, finite low half
        lambda b: b.fill_(NAN),                                 # all-NaN block
        lambda b: (b.__setitem__(2, INF), b[8:].fill_(NAN)),    # inf in one half, all-NaN other half
        lambda b: (b.__setitem__(9, -INF), b.__setitem__(1, NAN)),
        lambda b: b.__setitem__(14, INF),                       # inf, no NaN
        lambda b: b.fill_(-0.0),                                # -0.0 block
        lambda b: (b.zero_(), b.__setitem__(15, -0.0)),
        lambda b: b[:8].mul_(1e-30),                            # the block max sits in the high half
        lambda b: b[8:].mul_(1e4),
        lambda b: b[8:].mul_(1e35),                             # a finite scale above the window (inf in fp16)
    ]
    for k, j in enumerate(range(0, n_blocks, 5)):
        cases[k % len(cases)](x[j])
    return x


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
def test_grouped_nvfp4_equals_single_tensor_kernel(dtype):
    dev = torch.device("cuda")
    # whole tiles + a partial last tile, whole tiles only, a partial tile only, one whole tile
    sizes = [512 * 3 + 100, 512 * 2, 37, 512]
    xs = [_special_blocks(n, 7 + i).to(dtype).reshape(-1, 64 if n % 4 == 0 else 16).to(dev)
          for i, n in enumerate(sizes)]
    big = 1e30 if dtype != torch.float16 else 6e4
    # per slot: an in-range amax, one that puts the block scales above the exact-division window, a tiny one (scales
    # clamp at 448), and the tensor's own finite max
    amax = torch.tensor([8.0, big, 1e-3, float(xs[3].float().nan_to_num(0, 0, 0).abs().max())], device=dev)
    slot_of = [0, 1, 2, 3]
    want = [ops.fake_quant_nvfp4(x, amax[s:s + 1]) for x, s in zip(xs, slot_of)]

    ys = [torch.full_like(x, 7.0) for x in xs]
    ops.fake_quant_nvfp4_multi(ops.TensorTable(xs, slot_of, ys, "block16"), amax)
    for i, (y, w) in enumerate(zip(ys, want)):
        assert torch.equal(_bits(y), _bits(w)), f"fake_quant_nvfp4_multi, entry {i}"

    ys = [torch.full_like(x, 7.0) for x in xs]
    table = ops.TensorTable(xs, slot_of, ys, "block16", fused=True)
    slots = torch.zeros(4, dtype=torch.float32, device=dev)
    ops.collect_fake_quant_nvfp4_multi(table, slots, amax)
    for i, (y, w) in enumerate(zip(ys, want)):
        assert torch.equal(_bits(y), _bits(w)), f"collect_fake_quant_nvfp4_multi, entry {i}"
    ref_slots = ops.amax_per_tensor_multi_(torch.zeros(4, dtype=torch.float32, device=dev),
                                           ops.TensorTable(xs, slot_of, unit="vec32"))
    torch.cuda.synchronize()
    assert torch.equal(_bits(slots), _bits(ref_slots))

"""The grouped NVFP4 step at the sizes it runs at.  bench.py measures one graph step of ``ShardedPTQEngine(LLAMA3_8B,
4096 tokens, bf16)`` into a ring of 4 output buffers: 224 table entries, 5.1 G elements, 56 writers per buffer.  The
smaller grouped tests never reach the code that only such tables reach: the fix-up's later 256-entry rounds, descriptor
lookup over hundreds of entries and ~600 k CTAs, crowded rings of two entry sizes, tables of more than 2^32 elements.

Two references:
- the sequential engine (per-quantizer collect -> export -> ``fake_quant_nvfp4``), bit for bit after every step of a
  sequence that exercises the speculation (the fp32 arena, the exported amax and the full content of every output
  buffer; the fix-up's redo counter must count exactly the entries whose exported amax changed);
- the NumPy oracle (``o.fake_quant_nvfp4`` / ``o.reduce_amax``) on rows pulled to the host: the first and last rows of
  the entries whose output survives in each buffer, and the rows that hold the injected inf / NaN.

The ops-level tables check the grouped launches against their per-tensor kernels and the oracle, and the bench step's
activations are reused for one grouped amax and one grouped block-log2 histogram over more than 2^32 elements."""

import numpy as np
import pytest
import torch

from model_optimizer_b200 import ops
from model_optimizer_b200.engine import LLAMA3_8B, LLAMA3_70B, ModelPlan, ShardedPTQEngine
from oracle import oracle_np as o

pytestmark = pytest.mark.gpu

NAN, INF = float("nan"), float("inf")
DT = {torch.bfloat16: "bf16", torch.float16: "f16", torch.float32: "f32"}
# 560 entries, as LLAMA3_70B, with widths whose live bounds fall inside tiles at 40 tokens (640- and 1280-block
# entries).  Every LLAMA3_70B entry is a whole number of tiles (8192 / 16 = 512 blocks per token), so its tables never
# have fix-up pieces.
NARROW_80L = ModelPlan("narrow-80-layers", 256, 512, 80, 64)


def _bits(t):
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()])


def _host(t):
    return t.detach().float().cpu().numpy()


def _same(got, want, what):
    """bit-exact fp32 images, NaN positions included"""
    got, want = np.ascontiguousarray(got, np.float32), np.ascontiguousarray(want, np.float32)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    ok = (got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))
    if not ok.all():
        i = tuple(np.argwhere(~ok)[0])
        raise AssertionError(f"{what}: {int((~ok).sum())}/{ok.size} mismatches, first at {i}: got {got[i]!r} "
                             f"want {want[i]!r}")


def _need_free(gb):
    free, _ = torch.cuda.mem_get_info()
    if free < gb * 2 ** 30:
        pytest.skip(f"needs {gb} GB of free device memory, {free / 2 ** 30:.1f} GB free (a shared device)")


def _peak_check(base, limit):
    peak = torch.cuda.max_memory_allocated() - base
    print(f"peak allocated {peak / 1e9:.2f} GB")
    assert peak <= limit, f"{peak / 1e9:.2f} GB allocated, over the {limit / 1e9:.0f} GB budget"


# ---- the engine pair ------------------------------------------------------------------------------------------------
class _Pair:
    """The grouped engine and the sequential one over the SAME activations, each with its own outputs: a ring of
    ``n_ring`` buffers (``alloc_outputs``) or, for ``n_ring=None``, one buffer of exactly its size per quantizer."""

    def __init__(self, plan, tokens, dtype, n_ring, seed):
        self.tokens, self.dtype, self.n_ring = tokens, dtype, n_ring
        self.fused = ShardedPTQEngine(plan, tokens, "nvfp4", dtype, "cuda", grouped=True)
        self.ref = ShardedPTQEngine(plan, tokens, "nvfp4", dtype, "cuda", grouped=False)
        self.acts = self.fused.alloc_activations(seed=seed)
        self.cins = [cin for _, _, cin in self.fused.quantizers]
        self.n = len(self.acts)
        self.outs = []
        for eng in (self.fused, self.ref):
            outs = eng.alloc_outputs(n_ring) if n_ring else \
                [torch.empty(x.numel(), dtype=dtype, device="cuda") for x in self.acts]
            for b in outs:
                b.zero_()                # the tails of the ring are never written: start both sides equal
            eng.capture(self.acts, outs)
            self.outs.append(outs)
        (self.table,) = self.fused._graphs["tables"]
        idx = {name: i for i, name in enumerate(self.fused.arena.names())}
        self.slot = [idx[qn] for qn, _, _ in self.fused.quantizers]
        self.slots = torch.tensor(self.slot, device="cuda")
        self.samples = []                # (entry, output buffer, rows) checked against the oracle after every step
        self.run_max = {}                # per sampled entry: max |x| over the batches since the last reset

    def buffer_of(self, i):
        return i % self.n_ring if self.n_ring else i

    def close(self):
        """Drop every device buffer, including those a failure's traceback would keep alive through this object."""
        for eng in (self.fused, self.ref):
            eng._graphs, eng._graph_sets, eng._tables = {}, [], {}
        self.table._keep = None
        self.acts.clear()
        for outs in self.outs:
            outs.clear()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()

    def step(self, what, expect_redo):
        fused, ref = self.fused, self.ref
        before = _bits(ref.amax_arena[self.slots]).clone()
        r0 = int(fused.redo_count)
        fused.step_graph()
        ref.step_graph()
        torch.cuda.synchronize()
        changed = int((_bits(ref.amax_arena[self.slots]) != before).sum())
        assert torch.equal(_bits(fused.arena.freeze()), _bits(ref.arena.freeze())), f"{what}: fp32 arena"
        assert torch.equal(_bits(fused.amax_arena), _bits(ref.amax_arena)), f"{what}: exported amax"
        for k, (a, b) in enumerate(zip(*self.outs)):
            assert torch.equal(_bits(a), _bits(b)), f"{what}: output buffer {k}"
        assert int(fused.redo_count) - r0 == changed, f"{what}: redo count"
        assert changed == expect_redo, f"{what}: exported amaxes that changed"
        self.check_oracle(what)

    def reset(self):
        for eng in (self.fused, self.ref):
            eng.reset()
        self.run_max = {}

    def check_oracle(self, what):
        """the sampled rows' outputs against the oracle with the exported amax; the arena slot against the running max
        of the whole tensor, which torch reduces on the device"""
        arena = _host(self.fused.arena.freeze())
        exported = _host(self.fused.amax_arena)
        dt = DT[self.dtype]
        for i, b, rows in self.samples:
            x, cin, s = self.acts[i], self.cins[i], self.slot[i]
            batch, prev = float(x.abs().amax().float()), self.run_max.get(i, 0.0)
            self.run_max[i] = NAN if np.isnan(batch) or np.isnan(prev) else max(batch, prev)
            _same(arena[s:s + 1], np.float32([self.run_max[i]]), f"{what}: entry {i} amax")
            for r in rows:
                xr = _host(x[r])
                ra = float(o.reduce_amax(xr))
                assert np.isnan(arena[s]) if np.isnan(ra) else (np.isnan(arena[s]) or ra <= arena[s]), \
                    f"{what}: entry {i} row {r} amax"
                got = _host(self.outs[0][b][r * cin:(r + 1) * cin])
                _same(got, o.fake_quant_nvfp4(xr[None], np.float32(exported[s]), dt)[0],
                      f"{what}: entry {i} row {r} (buffer {b}) vs the oracle")


def _grow(acts, entries):
    for i in entries:
        x = acts[i].view(-1)
        x[7] = x.abs().max().float() * 4                     # a new unique maximum in row 0


def _put(acts, entry, row, col, value):
    acts[entry][row, col] = value


# ---- 1 + 2. the Llama-3-8B table --------------------------------------------------------------------------------------
def _llama8b_samples(pair):
    """Per output buffer, the entry written into it last (rows 0, last and a middle row that gets a special value) and,
    when that one is narrower, the last 14336-column entry of the buffer: its rows past every later writer's extent
    survive (from the first such row).  One buffer per quantizer: the entries of the first, a middle and the last layer
    and those the ring samples."""
    t, n, cins = pair.tokens, pair.n, pair.cins
    cmax = max(cins)
    mid = t // 2 + 1
    if pair.n_ring is None:
        entries = [*range(7), *range(112, 119), *range(217, 224), 202, 209, 216]
        return [(i, i, [0, t - 1, mid]) for i in entries]
    res = []
    for b in range(pair.n_ring):
        writers = [i for i in range(n) if i % pair.n_ring == b]
        last = writers[-1]
        res.append((last, b, [0, t - 1, mid]))
        if cins[last] < cmax:
            e = max(i for i in writers if cins[i] == cmax)
            r0 = -(-max(cins[i] for i in writers if i > e) * t // cmax)
            assert 0 < r0 < t - 2
            res.append((e, b, [r0, t - 1, (r0 + t) // 2]))
    return res


def _llama8b_sequence(pair):
    """first layer = entries 0..6, layer 16 = 112..118, last layer = 217..223; 202 / 209 / 216 are the down_proj
    entries of layers 28..30, whose tails survive in ring buffers 2 / 1 / 0"""
    n, acts = pair.n, pair.acts
    pair.step("from reset", n)
    pair.step("same batch again", 0)
    for x in acts:
        x.mul_(0.5)
    pair.step("lower batch", 0)
    subset = [1, 5, 114, 118, 202, 220, 223]
    _grow(acts, subset)
    pair.step("growth in a subset", len(subset))
    for i in subset:                                         # the unique maximum sits in row 0, a sampled row
        _same(_host(pair.fused.arena.freeze()[pair.slot[i]:pair.slot[i] + 1]),
              np.float32([o.reduce_amax(_host(acts[i][0]))]), f"growth: entry {i} amax vs the oracle")
    for x in acts:
        x.mul_(3)
    pair.step("growth in all tensors", n)
    rows = {i: r for i, _, (_, _, r) in pair.samples}
    mid = pair.tokens // 2 + 1
    specials = [(2, 5, INF), (4, 9, NAN), (116, 5, INF), (116, 100, NAN), (117, 3, -INF), (221, 17, NAN),
                (222, 33, -INF), (209, 40, INF), (216, 41, NAN)]
    for i, col, v in specials:
        _put(acts, i, rows.get(i, mid), col, v)
    pair.step("inf and NaN", len({i for i, _, _ in specials}))
    pair.step("inf and NaN again", 0)
    acts[0].zero_()
    pair.step("an all-zero tensor", 0)
    pair.reset()
    acts[1].zero_()
    pair.step("all-zero tensors from reset", n - 2)


def _grouped_stats_over(acts):
    """One grouped amax (vec32) and one grouped block-log2 histogram over every tensor of ``acts`` plus a zero-element
    entry, against one per-tensor launch each."""
    empty = torch.empty(0, 16, dtype=acts[0].dtype, device="cuda")
    xs = [*acts[:100], empty, *acts[100:]]
    try:
        _grouped_stats(xs, [*range(100), 0, *range(100, len(acts))], len(acts))
    finally:
        xs.clear()


def _grouped_stats(xs, slot_of, n_slots):
    assert sum(x.numel() for x in xs) > 2 ** 32
    want = torch.zeros(n_slots, device="cuda")
    for x, s in zip(xs, slot_of):
        if x.numel():
            ops.amax_per_tensor_(want[s:s + 1], x)
    got = ops.amax_per_tensor_multi_(torch.zeros(n_slots, device="cuda"), ops.TensorTable(xs, slot_of, unit="vec32"))
    torch.cuda.synchronize()
    assert torch.equal(_bits(got), _bits(want)), "grouped amax over the whole table"
    h_want = torch.zeros(n_slots, 512, dtype=torch.int64, device="cuda")
    m_want = torch.zeros(n_slots, device="cuda")
    for x, s in zip(xs, slot_of):
        if x.numel():
            ops.nvfp4_block_log2_hist_(h_want[s], m_want[s:s + 1], x)
    h = torch.zeros_like(h_want)
    m = torch.zeros_like(m_want)
    table = ops.TensorTable(xs, slot_of, unit="block16")
    assert table.n == len(xs) and table.total_ctas > 600_000
    ops.nvfp4_block_log2_hist_multi_(h, m, table)
    torch.cuda.synchronize()
    assert torch.equal(h, h_want), "grouped block-log2 histogram over the whole table"
    assert torch.equal(_bits(m), _bits(m_want)), "grouped running max over the whole table"
    assert int(h.sum()) > 0


def test_bench_step():
    """bench.py's step: LLAMA3_8B at 4096 tokens, bf16, a ring of 4 buffers; then the grouped amax and histogram over
    the same 5.1 G activations."""
    _need_free(16)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    pair = _Pair(LLAMA3_8B, 4096, torch.bfloat16, 4, seed=11)
    try:
        t = pair.table
        assert t.n == 224 == pair.n
        assert sum(x.numel() for x in pair.acts) > 2 ** 32
        assert t.fixup_bytes == 0 and t.n_pieces == 0          # every live bound is tile-aligned
        assert [sum(1 for i in range(pair.n) if i % 4 == b) for b in range(4)] == [56] * 4
        assert {pair.cins[i] for i in range(pair.n) if i % 4 == 0} == {4096, 14336}
        pair.samples = _llama8b_samples(pair)
        assert len(pair.samples) == 7                          # 4 last writers, 3 surviving 14336-column tails
        _llama8b_sequence(pair)
        _grouped_stats_over(pair.acts)
        _peak_check(base, 14e9)
    finally:
        pair.close()


def test_every_entry_of_llama8b():
    """LLAMA3_8B at 1024 tokens with one output buffer per quantizer: every entry's full output is compared."""
    _need_free(12)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    pair = _Pair(LLAMA3_8B, 1024, torch.bfloat16, None, seed=5)
    try:
        assert pair.table.n == 224 and pair.table.n_pieces == 0
        pair.samples = _llama8b_samples(pair)
        _llama8b_sequence(pair)
        _peak_check(base, 9e9)
    finally:
        pair.close()


# ---- 3. more than 512 entries: every 256-entry round of the fix-up -----------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32], ids=["bf16", "f16", "f32"])
@pytest.mark.parametrize("n_ring", [3, 4, 7, None], ids=["ring3", "ring4", "ring7", "one_per_quantizer"])
@pytest.mark.parametrize("plan", [LLAMA3_70B, NARROW_80L], ids=["llama70b", "narrow80"])
def test_fixup_rounds(plan, n_ring, dtype):
    pair = _Pair(plan, 40, dtype, n_ring, seed=29)
    try:
        n, acts, t = pair.n, pair.acts, pair.table
        assert t.n == n == 560 > 512
        if plan is NARROW_80L and n_ring in (3, 4):
            assert t.n_pieces > 0                              # live bounds inside tiles: the fix-up's pieces run
        else:                                                  # a ring of 7 gives each buffer one linear's entries
            assert t.n_pieces == 0
        # the last entry written into each buffer, first and last rows; one per quantizer: one entry of each round
        pair.samples = [(i, pair.buffer_of(i), [0, 39]) for i in
                        (range(n - n_ring, n) if n_ring else (0, 255, 256, 511, 512, 559))]
        pair.step("from reset", n)
        pair.step("same batch again", 0)
        for what, entries in [("growth only in entries >= 256", [256, 300, 441, 511, 557]),
                              ("growth only in entries >= 512", [512, 530, 559]),
                              ("growth only in entries < 256", [0, 100, 255]),
                              ("growth on both sides of 256", [255, 256])]:
            _grow(acts, entries)
            pair.step(what, len(entries))
        for x in acts:
            x.mul_(0.5)
        pair.step("lower batch", 0)
        for x in acts:
            x.mul_(3)
        pair.step("growth in all tensors", n)
        _put(acts, 10, 20, 5, INF)
        _put(acts, 300, 21, 9, NAN)
        _put(acts, 540, 22, 3, -INF)
        _put(acts, 558, 39, 7, NAN)
        pair.step("inf and NaN in every round", 4)
        pair.step("inf and NaN again", 0)
        acts[400].zero_()
        pair.step("an all-zero tensor", 0)
        pair.reset()
        acts[7].zero_()
        pair.step("all-zero tensors from reset", n - 2)
    finally:
        pair.close()


# ---- 4. grouped launches over large synthetic tables -------------------------------------------------------------------
# (rows, cols): 1, 511, 512, 513 and 1025 blocks; odd row counts
SHAPES = [(1, 16), (7, 1168), (1, 8192), (27, 304), (5, 3280), (3, 48)]
N_ENTRIES = 600
N_SLOTS = 400


def _synthetic(dtype, seed):
    """600 entries of mixed sizes with a zero-element entry at 333; entries 400.. share slots 0..49 with 4 others;
    values at scales 2^-6 .. 2^5, a few inf / NaN"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    xs = []
    for i in range(N_ENTRIES):
        shape = (0, 16) if i == 333 else SHAPES[i % len(SHAPES)]
        xs.append((torch.randn(shape, device="cuda", generator=g) * 2.0 ** (i % 12 - 6)).to(dtype))
    slot_of = [i if i < N_SLOTS else (i * 7) % 50 for i in range(N_ENTRIES)]
    xs[17].view(-1)[3] = INF
    xs[290].view(-1)[-1] = NAN
    xs[455].view(-1)[100] = -INF
    return xs, slot_of


def _per_slot_amax(xs, slot_of):
    want = torch.zeros(N_SLOTS, device="cuda")
    for x, s in zip(xs, slot_of):
        if x.numel():
            ops.amax_per_tensor_(want[s:s + 1], x)
    return want


def _oracle_slot_amax(xs, slot_of):
    want = np.zeros(N_SLOTS, np.float32)
    for x, s in zip(xs, slot_of):
        if x.numel():
            a = o.reduce_amax(_host(x))
            want[s] = np.float32(np.nan) if np.isnan(a) or np.isnan(want[s]) else max(want[s], a)
    return want


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32], ids=["bf16", "f16", "f32"])
def test_synthetic_table_amax_and_hist(dtype):
    xs, slot_of = _synthetic(dtype, 41)
    table = ops.TensorTable(xs, slot_of, unit="vec32")
    assert table.n == N_ENTRIES
    want = _per_slot_amax(xs, slot_of)
    got = ops.amax_per_tensor_multi_(torch.zeros(N_SLOTS, device="cuda"), table)
    torch.cuda.synchronize()
    assert torch.equal(_bits(got), _bits(want))
    _same(_host(got), _oracle_slot_amax(xs, slot_of), "grouped amax vs the oracle")

    h = torch.zeros(N_SLOTS, 512, dtype=torch.int64, device="cuda")
    m = torch.zeros(N_SLOTS, device="cuda")
    ops.nvfp4_block_log2_hist_multi_(h, m, ops.TensorTable(xs, slot_of, unit="block16"))
    h_want, m_want = torch.zeros_like(h), torch.zeros_like(m)
    for x, s in zip(xs, slot_of):
        if x.numel():
            ops.nvfp4_block_log2_hist_(h_want[s], m_want[s:s + 1], x)
    torch.cuda.synchronize()
    assert torch.equal(h, h_want)
    assert torch.equal(_bits(m), _bits(m_want))
    h_o = np.zeros((N_SLOTS, 512), np.int64)
    for x, s in zip(xs, slot_of):
        if x.numel():
            h_o[s] += o.nvfp4_block_log2_hist(_host(x))[0]
    assert np.array_equal(h.cpu().numpy(), h_o), "grouped block-log2 histogram vs the oracle"


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32], ids=["bf16", "f16", "f32"])
def test_synthetic_table_fake_quant(dtype):
    xs, slot_of = _synthetic(dtype, 43)
    amax = ops.amax_export(_per_slot_amax(xs, slot_of), dtype)
    ys = [torch.full_like(x, 7.0) for x in xs]
    ops.fake_quant_nvfp4_multi(ops.TensorTable(xs, slot_of, ys, "block16"), amax)
    torch.cuda.synchronize()
    amax_h = _host(amax)
    for i, (x, y, s) in enumerate(zip(xs, ys, slot_of)):
        if x.numel():
            assert torch.equal(_bits(y), _bits(ops.fake_quant_nvfp4(x, amax[s:s + 1]))), f"entry {i}"
            _same(_host(y), o.fake_quant_nvfp4(_host(x), amax_h[s], DT[dtype]), f"entry {i} vs the oracle")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32], ids=["bf16", "f16", "f32"])
def test_synthetic_table_fused_step(dtype):
    """entries 0..399 write prefixes of 8 shared buffers in turn (50 writers each, live bounds inside tiles), the rest
    a buffer each; collect + fix-up + export against per-tensor amax, export and fake quant launches in table order"""
    xs, slot_of = _synthetic(dtype, 47)
    cap = max(x.numel() for x in xs)
    shared = [torch.zeros(cap, dtype=dtype, device="cuda") for _ in range(8)]
    own = [torch.zeros(x.numel(), dtype=dtype, device="cuda") for x in xs[400:]]
    bufs = shared + own
    buf_of = [i % 8 if i < 400 else 8 + i - 400 for i in range(N_ENTRIES)]
    ys = [bufs[b][: x.numel()].view_as(x) for x, b in zip(xs, buf_of)]
    table = ops.TensorTable(xs, slot_of, ys, "block16", fused=True)
    assert table.n == N_ENTRIES and table.n_pieces > 0 and len(table.passes) == 2
    slots = torch.zeros(N_SLOTS, device="cuda")
    amax = torch.zeros(N_SLOTS, dtype=dtype, device="cuda")
    redo = torch.zeros(1, dtype=torch.int32, device="cuda")
    ref_slots = torch.zeros(N_SLOTS, device="cuda")
    last_writer = {b: i for i, b in enumerate(buf_of) if xs[i].numel()}
    for rnd, grow in enumerate([[], [], [3, 300, 445, 599], [250, 260, 520]]):
        for i in grow:                                         # 4 x the slot's amax: above every entry sharing it
            xs[i].view(-1)[7] = ref_slots[slot_of[i]] * 4
        old = _bits(amax).clone()
        r0 = int(redo)
        ops.collect_fake_quant_nvfp4_multi(table, slots, amax)
        ops.fake_quant_nvfp4_multi_fixup(table, slots, amax, redo)
        amax.copy_(ops.amax_export(slots, dtype))
        for x, s in zip(xs, slot_of):
            if x.numel():
                ops.amax_per_tensor_(ref_slots[s:s + 1], x)
        want = [torch.zeros_like(b) for b in bufs]
        for x, b, s in zip(xs, buf_of, slot_of):
            if x.numel():
                want[b][: x.numel()] = ops.fake_quant_nvfp4(x, amax[s:s + 1]).view(-1)
        torch.cuda.synchronize()
        assert torch.equal(_bits(slots), _bits(ref_slots)), f"round {rnd}: slots"
        for k, (a, w) in enumerate(zip(bufs, want)):
            assert torch.equal(_bits(a), _bits(w)), f"round {rnd}: output buffer {k}"
        changed = (_bits(amax) != old)[torch.tensor(slot_of, device="cuda")]
        assert int(redo) - r0 == int(changed.sum()), f"round {rnd}: redo count"
        if rnd == 1:
            assert int(changed.sum()) == 0
        if rnd >= 2:                                           # every entry sharing a grown slot is redone
            assert int(changed.sum()) == sum(1 for s in slot_of if s in {slot_of[i] for i in grow})
    for b, i in last_writer.items():                           # the last writer's whole output survives
        _same(_host(bufs[b][: xs[i].numel()]).reshape(xs[i].shape),
              o.fake_quant_nvfp4(_host(xs[i]), np.float32(float(amax[slot_of[i]])), DT[dtype]),
              f"entry {i} (buffer {b}) vs the oracle")

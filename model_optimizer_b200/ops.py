"""Tensor-level wrappers over the C-ABI (``include/b200quant.h``).

PyTorch is plumbing here: device memory, the current stream and dtype tags.  Every function
takes CUDA tensors and enqueues exactly one kernel family on ``torch.cuda.current_stream()``;
CPU tensors raise -- there is no fallback path.
"""

from __future__ import annotations

import bisect
import functools

import torch

from . import _lib
from ._lib import BF16, F16, F32, B200QuantError, call

_DT = {torch.float32: F32, torch.float16: F16, torch.bfloat16: BF16}


def _dt(t: torch.Tensor) -> int:
    try:
        return _DT[t.dtype]
    except KeyError:
        raise B200QuantError(f"unsupported dtype {t.dtype} (float32 / float16 / bfloat16 only)") from None


def _prep(t: torch.Tensor, name: str = "tensor") -> torch.Tensor:
    if not t.is_cuda:
        raise B200QuantError(f"{name} must be a CUDA tensor: the b200 engine has no CPU fallback")
    return t if t.is_contiguous() else t.contiguous()


def _stream(t: torch.Tensor) -> int:
    return torch.cuda.current_stream(t.device).cuda_stream


def _slots(t: torch.Tensor, name: str = "slots") -> torch.Tensor:
    if t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous():
        raise B200QuantError(f"{name} must be a contiguous float32 CUDA tensor")
    return t


# ------------------------------------------------------------------------------------------------
# calibration collect
# ------------------------------------------------------------------------------------------------
def amax_per_tensor_(slot: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """slot[0] = max(slot[0], max|x|)  (fp32 slot; NaN propagates)."""
    x = _prep(x, "x")
    _slots(slot, "slot")
    call("b200q_amax_per_tensor", x.data_ptr(), _dt(x), x.numel(), slot.data_ptr(), _stream(x))
    return slot


def amax_rows_(slots: torch.Tensor, x: torch.Tensor, row_len: int) -> torch.Tensor:
    """x viewed as [numel/row_len, row_len]; slots[r % slots.numel()] = max(., max_j |x[r, j]|)."""
    x = _prep(x, "x")
    _slots(slots)
    n_rows = x.numel() // row_len if row_len else 0
    if n_rows * row_len != x.numel():
        raise B200QuantError("x.numel() is not a multiple of row_len")
    call("b200q_amax_rows", x.data_ptr(), _dt(x), n_rows, row_len, slots.numel(), slots.data_ptr(), _stream(x))
    return slots


def amax_cols_(slots: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """x viewed as [-1, C] with C = slots.numel(); slots[c] = max(., max_r |x[r, c]|)."""
    x = _prep(x, "x")
    _slots(slots)
    c = slots.numel()
    call("b200q_amax_cols", x.data_ptr(), _dt(x), x.numel() // c, c, slots.data_ptr(), _stream(x))
    return slots


def abssum_cols_(slots: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    x = _prep(x, "x")
    _slots(slots)
    c = slots.numel()
    call("b200q_abssum_cols", x.data_ptr(), _dt(x), x.numel() // c, c, slots.data_ptr(), _stream(x))
    return slots


HIST_SCRATCH_ELEMS = 32768 + 160 * 1536      # B200Q_HIST_SCRATCH_ELEMS (include/b200quant.h)


def hist_scratch(device) -> torch.Tensor:
    """Zeroed int32 scratch for the 16-bit pattern-counting path of ``histogram_`` / ``histogram_planned_``
    (32768 atomic pattern counters + one 1536-word row per CTA)."""
    return torch.zeros(HIST_SCRATCH_ELEMS, dtype=torch.int32, device=device)


def _check_scratch(scratch):
    if scratch is not None and (scratch.dtype != torch.int32 or scratch.numel() != HIST_SCRATCH_ELEMS or not scratch.is_cuda
                                or not scratch.is_contiguous()):
        raise B200QuantError(f"scratch must be a contiguous int32 CUDA tensor of {HIST_SCRATCH_ELEMS} elements (ops.hist_scratch)")


def histogram_(hist: torch.Tensor, x: torch.Tensor, range_max: torch.Tensor, take_abs: bool = True,
               scratch: torch.Tensor | None = None) -> torch.Tensor:
    """hist[bin] += count with torch.histc(bins=hist.numel(), min=0, max=range_max) binning.  ``scratch``: see
    ``histogram_planned_``.  ``range_max == 0`` counts the zeros in bin ``nbins // 2``, where histc puts them when every
    value is zero (it widens the empty range to [-1, 1]).  Non-zero values are outside [0, 0] and skipped; histc would
    instead bin them over the data's own min and max, which this one-pass kernel does not know."""
    x = _prep(x, "x")
    _slots(hist, "hist")
    _slots(range_max, "range_max")
    _check_scratch(scratch)
    call("b200q_histogram_ex", x.data_ptr(), _dt(x), x.numel(), int(take_abs), range_max.data_ptr(), hist.numel(), None,
         hist.data_ptr(), None if scratch is None else scratch.data_ptr(), _stream(x))
    return hist


def live_block_ranges(inputs, outputs, block_bytes: int) -> list[tuple[int, int]]:
    """For a table whose entries run in order, entry i reading ``inputs[i]`` and writing ``outputs[i]`` (both
    ``(address, nbytes)``), per entry ``(live_from, contested_to)`` in ``block_bytes`` blocks of its output:
    ``live_from`` is the first block that no LATER entry writes, so blocks ``[live_from, n)`` are the ones the entry
    leaves in the buffer and the live ranges of all entries are disjoint; ``[live_from, contested_to)`` is the part of
    that range an EARLIER entry writes too.  One grid over the table runs the entries concurrently, so that part may end
    up holding the earlier entry's result; rewriting it afterwards (and all of ``[live_from, n)`` for an entry whose
    result changed) leaves every output buffer as running the entries in order leaves it.  Raises
    :class:`B200QuantError` when an output overlaps any input, or two outputs overlap without starting at the same
    address (a later output must cover a prefix of an earlier one)."""
    if len(inputs) != len(outputs):
        raise B200QuantError("one output per input")
    spans = sorted((a, a + n) for a, n in inputs if n > 0)
    starts = [s for s, _ in spans]
    reach, r = [], 0                                   # reach[k]: largest end among the first k + 1 inputs by start
    for _, e in spans:
        r = max(r, e)
        reach.append(r)
    for a, n in outputs:
        k = bisect.bisect_left(starts, a + n)          # inputs starting below the output's end
        if n > 0 and k > 0 and reach[k - 1] > a:
            raise B200QuantError("fused collect + fake quant: an output overlaps an input")
    ends = {}                                          # output base address -> largest extent
    for a, n in outputs:
        if n > 0:
            ends[a] = max(ends.get(a, a), a + n)
    r = 0
    for a in sorted(ends):
        if a < r:
            raise B200QuantError("fused collect + fake quant: outputs overlap without sharing a base address")
        r = max(r, ends[a])
    live, after = [0] * len(outputs), {}               # after[base]: blocks written by the entries after i
    for i in range(len(outputs) - 1, -1, -1):
        a, n = outputs[i]
        live[i] = min(n // block_bytes, after.get(a, 0))
        after[a] = max(after.get(a, 0), n // block_bytes)
    ranges, before = [], {}                            # before[base]: blocks written by the entries before i
    for i, (a, n) in enumerate(outputs):
        ranges.append((live[i], max(live[i], min(n // block_bytes, before.get(a, 0)))))
        before[a] = max(before.get(a, 0), n // block_bytes)
    return ranges


NVFP4_TILE_BLOCKS = 512                                # one CTA tile of the NVFP4 grids: 256 threads x 2 blocks


def output_tiles(outputs, block_bytes: int, tile_blocks: int = NVFP4_TILE_BLOCKS):
    """Store-order bookkeeping of the fused collect + fake quant over ``outputs`` (``(address, nbytes)`` per entry, the
    layouts ``live_block_ranges`` accepts).  Outputs sharing a buffer are prefixes of it, so tile k (``tile_blocks``
    blocks of ``block_bytes``) of every entry writing that buffer covers the same bytes.  Buffer tiles are numbered
    buffer by buffer, in order of first use.  Returns ``(tile0, owner, expected, preflag, pieces)``:

    - ``tile0[i]``: the number of entry i's tile 0;
    - per buffer tile: ``owner``, the last entry writing any part of it (the one that leaves its first block);
      ``expected``, the number of earlier entries writing any part of it; ``preflag``, whether live blocks of more
      than one entry lie in it (a live bound inside the tile) -- its stores cannot be ordered by one check;
    - ``pieces``: ``(entry, from, to)`` block ranges, the live blocks of each entry inside a pre-flagged tile."""
    nblk = [n // block_bytes for _, n in outputs]
    live_from, after = [0] * len(outputs), {}          # as in live_block_ranges
    for i in range(len(outputs) - 1, -1, -1):
        a = outputs[i][0]
        live_from[i] = min(nblk[i], after.get(a, 0))
        after[a] = max(after.get(a, 0), nblk[i])
    bases = {}
    for i, (a, _) in enumerate(outputs):
        bases.setdefault(a, []).append(i)
    first = {}
    total = 0
    for a, ents in bases.items():
        first[a] = total
        total += -(-max(nblk[i] for i in ents) // tile_blocks)
    tile0 = [first[a] for a, _ in outputs]
    owner, expected, n_live = [-1] * total, [0] * total, [0] * total
    for a, ents in bases.items():
        ns = sorted(nblk[i] for i in ents)
        for k in range(-(-ns[-1] // tile_blocks)):
            # entries writing any block of tile k: those with more than k * tile_blocks blocks
            expected[first[a] + k] = len(ns) - bisect.bisect_right(ns, k * tile_blocks) - 1
    for i, lf in enumerate(live_from):
        if lf >= nblk[i]:
            continue
        t0, t1 = lf // tile_blocks, (nblk[i] - 1) // tile_blocks
        for k in range(-(-lf // tile_blocks), t1 + 1):          # tiles whose first block entry i leaves
            owner[tile0[i] + k] = i
        for k in {t0, t1}:                                       # only a range's end tiles can hold other live blocks
            n_live[tile0[i] + k] += 1
    preflag = [c > 1 for c in n_live]
    pieces = []
    for i, lf in enumerate(live_from):
        if lf >= nblk[i]:
            continue
        for k in sorted({lf // tile_blocks, (nblk[i] - 1) // tile_blocks}):
            if preflag[tile0[i] + k]:
                pieces.append((i, max(lf, k * tile_blocks), min(nblk[i], (k + 1) * tile_blocks)))
    return tile0, owner, expected, preflag, pieces


def second_pass_tiles(outputs, block_bytes: int, tile_blocks: int = NVFP4_TILE_BLOCKS) -> list[tuple[int, int]]:
    """The two-pass order of the fused collect + fake quant over ``outputs`` (as for ``output_tiles``): per entry the
    range ``[k_from, k_to)`` of its tiles that run in the SECOND pass -- the tiles it writes last while an earlier entry
    writes them too.  Every other tile runs in the first pass.  The second pass starts after the first has completed,
    and no two of its tiles cover the same bytes, so every tile ends with its last writer's stores; only the live
    blocks of other entries inside a pre-flagged tile (``output_tiles``) can still end wrong, and the fix-up rewrites
    them."""
    tile0, owner, expected, _, _ = output_tiles(outputs, block_bytes, tile_blocks)
    res = []
    for i, (_, n) in enumerate(outputs):
        n_tiles = -(-(n // block_bytes) // tile_blocks)
        k = 0
        while k < n_tiles and owner[tile0[i] + k] != i:      # the tiles an entry writes last are a suffix of its tiles
            k += 1
        k_to = k
        while k_to < n_tiles and expected[tile0[i] + k_to] > 0:   # ... and those with earlier writers a prefix
            k_to += 1
        res.append((k, k_to))
    return res


class TensorTable:
    """Device descriptor table for the multi-tensor launches (``b200q_amax_per_tensor_multi`` /
    ``b200q_fake_quant_nvfp4_multi``): build once per set of (static) buffers, launch many times -- e.g. inside a
    CUDA graph.  ``xs`` (and ``ys``): contiguous CUDA tensors of one dtype, 32-byte aligned; ``slots``: the amax slot
    index of each tensor.  ``fused`` (NVFP4 with ``ys``): a table for ``collect_fake_quant_nvfp4_multi`` /
    ``fake_quant_nvfp4_multi_fixup``, which also ships each entry's live output range (``live_block_ranges``) and
    refuses buffers those launches cannot reproduce the sequential result on."""

    def __init__(self, xs, slots=None, ys=None, unit: str = "vec32", fused: bool = False):
        if not xs:
            raise B200QuantError("empty tensor list")
        if fused and (ys is None or unit != "block16"):
            raise B200QuantError("a fused table needs outputs and unit='block16'")
        self.dtype = xs[0].dtype
        self.unit = unit
        self.device = xs[0].device
        es = xs[0].element_size()
        per_cta = 1024 if unit == "vec32" else 512                 # amax: 256 thr x 4 vectors; NVFP4: 256 thr x 2 blocks
        rows, first = [], 0
        for i, x in enumerate(xs):
            y = ys[i] if ys is not None else None
            if x.dtype != self.dtype or not x.is_cuda or not x.is_contiguous() or x.data_ptr() % 32:
                raise B200QuantError("multi-tensor launch: contiguous, 32-byte aligned CUDA tensors of one dtype")
            if y is not None and (y.dtype != x.dtype or y.numel() != x.numel() or not y.is_contiguous() or y.data_ptr() % 32):
                raise B200QuantError("multi-tensor launch: outputs must match the inputs")
            if unit == "vec32":
                if (x.numel() * es) % 32:
                    raise B200QuantError("multi-tensor amax: numel * itemsize must be a multiple of 32 bytes")
                n_units = x.numel() * es // 32
            else:
                if x.shape[-1] % 16:
                    raise B200QuantError("multi-tensor NVFP4: the last dim must be a multiple of 16")
                n_units = x.numel() // 16
            rows.append([x.data_ptr(), 0 if y is None else y.data_ptr(), n_units, first,
                         i if slots is None else int(slots[i])])
            first += (n_units + per_cta - 1) // per_cta
        self.total_ctas = first
        self.n = len(rows)
        self.max_slot = max(r[4] for r in rows)
        self.table = torch.tensor(rows, dtype=torch.int64).to(self.device)
        self.live = None
        if fused:
            nb = [x.numel() * es for x in xs]
            outputs = [(y.data_ptr(), n) for y, n in zip(ys, nb)]
            live = live_block_ranges([(x.data_ptr(), n) for x, n in zip(xs, nb)], outputs, 16 * es)
            _, _, _, _, pieces = output_tiles(outputs, 16 * es)
            self.live = torch.tensor(live, dtype=torch.int64).to(self.device)
            # the fused step runs as two passes over sub-tensor descriptors of the same entries (second_pass_tiles)
            tile_b = per_cta * 16 * es
            passes = ([], [])
            for (x, y, n_units, _, slot), (k0, k1) in zip(rows, second_pass_tiles(outputs, 16 * es)):
                n_t = (n_units + per_cta - 1) // per_cta
                for p, a, b in ((0, 0, k0), (1, k0, k1), (0, k1, n_t)):
                    if b > a:
                        passes[p].append([x + a * tile_b, y + a * tile_b, min(n_units, b * per_cta) - a * per_cta, 0,
                                          slot])
            self.passes = []
            for r in passes:
                first = 0
                for row in r:
                    row[3] = first
                    first += (row[2] + per_cta - 1) // per_cta
                if r:
                    self.passes.append((torch.tensor(r, dtype=torch.int64).to(self.device), len(r), first))
            self.n_pieces = len(pieces)
            self.pieces = torch.tensor(pieces or [(0, 0, 0)], dtype=torch.int64).to(self.device)
            # bytes the fix-up moves when no amax changes: the live blocks of the pre-flagged tiles are read and
            # written again
            self.fixup_bytes = sum(b - a for _, a, b in pieces) * 16 * es * 2
        self._keep = (list(xs), None if ys is None else list(ys))  # the table holds raw pointers


def amax_per_tensor_multi_(slots: torch.Tensor, table: TensorTable) -> torch.Tensor:
    """slots[table slot of tensor i] = max(., max|x_i|) for every tensor of the table, ONE launch."""
    _slots(slots)
    with torch.cuda.device(table.device):
        call("b200q_amax_per_tensor_multi", table.table.data_ptr(), table.n, table.total_ctas, _DT[table.dtype],
             slots.data_ptr(), torch.cuda.current_stream(table.device).cuda_stream)
    return slots


def fake_quant_nvfp4_multi(table: TensorTable, amax_base: torch.Tensor):
    """y_i = NVFP4 dynamic fake quant of x_i with global amax ``amax_base[slot_i]``, ONE launch."""
    if not amax_base.is_cuda or not amax_base.is_contiguous() or amax_base.dtype not in _DT:
        raise B200QuantError("amax_base must be a contiguous CUDA tensor (fp32 / fp16 / bf16)")
    with torch.cuda.device(table.device):
        call("b200q_fake_quant_nvfp4_multi", table.table.data_ptr(), table.n, table.total_ctas, _DT[table.dtype],
             amax_base.data_ptr(), _DT[amax_base.dtype], torch.cuda.current_stream(table.device).cuda_stream)


def _fused_args(table: TensorTable, slots: torch.Tensor, amax_base: torch.Tensor):
    if table.live is None:
        raise B200QuantError("the table was not built with fused=True")
    _slots(slots)
    if not amax_base.is_cuda or not amax_base.is_contiguous() or amax_base.dtype not in _DT:
        raise B200QuantError("amax_base must be a contiguous CUDA tensor (fp32 / fp16 / bf16)")


def collect_fake_quant_nvfp4_multi(table: TensorTable, slots: torch.Tensor, amax_base: torch.Tensor):
    """``fake_quant_nvfp4_multi(table, amax_base)`` and ``amax_per_tensor_multi_(slots, table)`` in ONE read of every
    input: the outputs are SPECULATIVE (quantized with the amax ``amax_base`` holds now, i.e. the previous export) until
    ``fake_quant_nvfp4_multi_fixup`` has run.  ``table``: built with ``fused=True``.  Two launches in stream order
    (``second_pass_tiles``): the second stores the tiles that entries sharing an output buffer write last."""
    _fused_args(table, slots, amax_base)
    with torch.cuda.device(table.device):
        for descs, n, total_ctas in table.passes:
            call("b200q_collect_fake_quant_nvfp4_multi", descs.data_ptr(), n, total_ctas, _DT[table.dtype],
                 slots.data_ptr(), amax_base.data_ptr(), _DT[amax_base.dtype],
                 torch.cuda.current_stream(table.device).cuda_stream)


def fake_quant_nvfp4_multi_fixup(table: TensorTable, slots: torch.Tensor, amax_base: torch.Tensor,
                                 redo_count: torch.Tensor):
    """Between ``collect_fake_quant_nvfp4_multi`` and the export of ``slots`` into ``amax_base``: redo, with the new
    amax, the live output range (``live_block_ranges``) of every entry whose exported amax is about to change, and
    rewrite the live blocks of the pre-flagged output tiles (``output_tiles``), so that after the export everything is
    bit-identical to collect -> export -> fake quant.  ``redo_count`` (int32 CUDA scalar) += number of entries redone."""
    _fused_args(table, slots, amax_base)
    if redo_count.dtype != torch.int32 or not redo_count.is_cuda or redo_count.numel() != 1:
        raise B200QuantError("redo_count must be an int32 CUDA tensor of one element")
    with torch.cuda.device(table.device):
        call("b200q_fake_quant_nvfp4_multi_fixup", table.table.data_ptr(), table.live.data_ptr(), table.n,
             _DT[table.dtype], slots.data_ptr(), amax_base.data_ptr(), _DT[amax_base.dtype], table.pieces.data_ptr(),
             table.n_pieces, redo_count.data_ptr(), torch.cuda.current_stream(table.device).cuda_stream)


def hist_plan_(plan_state: torch.Tensor, batch_amax: torch.Tensor, nbins0: int, capacity: int) -> torch.Tensor:
    """Device-side range planning of HistogramCalibrator.collect (no host sync): updates the 8-word plan state
    (upper, width, xmax_grow as fp32; nbins, initialized, overflow, n_growths as int32) for a batch whose |x| max
    is ``batch_amax`` (fp32 device scalar)."""
    if plan_state.dtype != torch.int32 or plan_state.numel() != 8 or not plan_state.is_cuda:
        raise B200QuantError("plan_state must be an int32 CUDA tensor of 8 elements")
    _slots(batch_amax, "batch_amax")
    call("b200q_hist_plan", batch_amax.data_ptr(), int(nbins0), int(capacity), plan_state.data_ptr(),
         _stream(plan_state))
    return plan_state


def histogram_planned_(hist: torch.Tensor, x: torch.Tensor, plan_state: torch.Tensor, take_abs: bool = True,
                       scratch: torch.Tensor | None = None):
    """hist[bin] += counts with the (nbins, upper) currently held by ``plan_state`` (see ``hist_plan_``).  ``scratch``
    (``hist_scratch(device)``; its counter part is left zeroed) enables the pattern-counting fast path for 16-bit
    inputs."""
    x = _prep(x, "x")
    _slots(hist, "hist")
    _check_scratch(scratch)
    call("b200q_histogram_ex", x.data_ptr(), _dt(x), x.numel(), int(take_abs), None, 0, plan_state.data_ptr(),
         hist.data_ptr(), None if scratch is None else scratch.data_ptr(), _stream(x))
    return hist


def hist_search_percentile(hist: torch.Tensor, percentile: float) -> torch.Tensor:
    """-> int32 device scalar: searchsorted(cumsum(hist / total), percentile / 100)."""
    _slots(hist, "hist")
    idx = torch.empty(1, dtype=torch.int32, device=hist.device)
    call("b200q_hist_search_percentile", hist.data_ptr(), hist.numel(), float(percentile), idx.data_ptr(), _stream(hist))
    return idx


def hist_search_entropy(hist: torch.Tensor, num_quant_bins: int, stride: int = 1, start_bin: int = 128) -> torch.Tensor:
    """-> fp64 KL divergence of every candidate threshold range(start_bin, nbins + 1, stride)."""
    _slots(hist, "hist")
    n = hist.numel()
    prefix = torch.empty(n + 1, dtype=torch.int64, device=hist.device)
    nz = torch.empty(n + 1, dtype=torch.int32, device=hist.device)
    div = torch.empty((n - start_bin) // stride + 1, dtype=torch.float64, device=hist.device)
    call("b200q_hist_search_entropy", hist.data_ptr(), n, int(num_quant_bins), int(stride), int(start_bin),
         prefix.data_ptr(), nz.data_ptr(), div.data_ptr(), _stream(hist))
    return div


def hist_search_mse(hist: torch.Tensor, centers: torch.Tensor, num_bits: int, unsigned: bool = False, stride: int = 1,
                    start_bin: int = 128) -> torch.Tensor:
    """-> fp32 loss of every candidate range(start_bin, len(centers), stride); num_bits 0 = FP8-E4M3."""
    _slots(hist, "hist")
    _slots(centers, "centers")
    n = centers.numel()
    if hist.numel() < n:
        raise B200QuantError("hist is shorter than centers")
    out = torch.empty((n - 1 - start_bin) // stride + 1, dtype=torch.float32, device=hist.device)
    call("b200q_hist_search_mse", hist.data_ptr(), centers.data_ptr(), n, int(num_bits), int(bool(unsigned)),
         int(stride), int(start_bin), out.data_ptr(), _stream(hist))
    return out


def nvfp4_block_log2_hist_(hist: torch.Tensor, running_max: torch.Tensor, x: torch.Tensor,
                           log2_min: float = -40.0, log2_max: float = 40.0) -> torch.Tensor:
    """hist (int64) += bincount of the log2 bin of every 16-element block amax; running_max = max(., amax)."""
    x = _prep(x, "x")
    _slots(running_max, "running_max")
    if hist.dtype != torch.int64 or not hist.is_cuda or not hist.is_contiguous():
        raise B200QuantError("hist must be a contiguous int64 CUDA tensor")
    if x.shape[-1] % 16 != 0:
        raise B200QuantError("last dim must be a multiple of 16 (pad with zeros first)")
    call("b200q_nvfp4_block_log2_hist", x.data_ptr(), _dt(x), x.numel() // 16, float(log2_min), float(log2_max),
         hist.numel(), hist.data_ptr(), running_max.data_ptr(), _stream(x))
    return hist


def nvfp4_block_log2_hist_multi_(hist: torch.Tensor, running_max: torch.Tensor, table: TensorTable,
                                 log2_min: float = -40.0, log2_max: float = 40.0) -> torch.Tensor:
    """``nvfp4_block_log2_hist_(hist[slot_i], running_max[slot_i : slot_i + 1], x_i)`` for every tensor of ``table``
    (built with ``unit="block16"``) in ONE launch: ``hist`` is the int64 ``[n_slots, nbins]`` table, ``running_max``
    the fp32 ``[n_slots]`` slots; entries that share a slot accumulate into it."""
    _slots(running_max, "running_max")
    if hist.dtype != torch.int64 or not hist.is_cuda or not hist.is_contiguous() or hist.dim() != 2:
        raise B200QuantError("hist must be a contiguous int64 CUDA tensor [n_slots, nbins]")
    if table.unit != "block16":
        raise B200QuantError("the table must be built with unit='block16'")
    if running_max.numel() != hist.shape[0] or table.max_slot >= hist.shape[0] or hist.device != table.device \
            or running_max.device != table.device:
        raise B200QuantError(f"hist / running_max must have a row per slot on {table.device} (largest slot "
                             f"{table.max_slot}, {hist.shape[0]} rows)")
    with torch.cuda.device(table.device):
        call("b200q_nvfp4_block_log2_hist_multi", table.table.data_ptr(), table.n, table.total_ctas, _DT[table.dtype],
             float(log2_min), float(log2_max), hist.shape[1], hist.data_ptr(), running_max.data_ptr(),
             torch.cuda.current_stream(table.device).cuda_stream)
    return hist


def reduce_keep_(x, n_outer, n_groups, rows_per_group, n_cols, max_slots=None, min_slots=None, sum_slots=None):
    """Signed max / min / sum over (outer, rows) of x viewed as [n_outer, n_groups, rows_per_group, n_cols]; the
    fp32 slots ([n_groups * n_cols], running) are updated in place."""
    x = _prep(x, "x")
    if x.numel() != n_outer * n_groups * rows_per_group * n_cols:
        raise ValueError("view does not cover the tensor")
    ptr = lambda t: None if t is None else _slots(t).data_ptr()  # noqa: E731
    call("b200q_reduce_keep", x.data_ptr(), _dt(x), n_outer, n_groups, rows_per_group, n_cols, ptr(max_slots),
         ptr(min_slots), ptr(sum_slots), _stream(x))


def amax_export(slots: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """fp32 slots -> tensor of ``dtype`` (the reference keeps ``_amax`` in the input dtype)."""
    _slots(slots)
    if dtype == torch.float32:
        return slots.clone()
    out = torch.empty(slots.shape, dtype=dtype, device=slots.device)
    call("b200q_amax_export", slots.data_ptr(), slots.numel(), out.data_ptr(), _DT[dtype], _stream(slots))
    return out


# ------------------------------------------------------------------------------------------------
# fake quant
# ------------------------------------------------------------------------------------------------
def _amax_arg(amax: torch.Tensor, like: torch.Tensor) -> torch.Tensor:
    if not amax.is_cuda:
        amax = amax.to(like.device)
    if amax.dtype not in _DT:
        amax = amax.float()
    return amax if amax.is_contiguous() else amax.contiguous()


def _out_arg(out, x: torch.Tensor) -> torch.Tensor:
    """``out`` (or a new tensor like ``x`` when None), refused unless the kernel can write all of x's elements to it."""
    if out is None:
        return torch.empty_like(x)
    if not isinstance(out, torch.Tensor) or out.device != x.device or out.dtype != x.dtype or out.shape != x.shape \
            or not out.is_contiguous():
        raise B200QuantError(f"out must be a contiguous {x.dtype} tensor of shape {tuple(x.shape)} on {x.device}")
    return out


def fake_quant_int(x, amax, num_bits=8, unsigned=False, narrow_range=True, outer=1, out=None):
    """Integer fake quant; ``amax[(i // outer) % amax.numel()]`` scales element i."""
    x = _prep(x, "x")
    amax = _amax_arg(amax, x)
    y = _out_arg(out, x)
    call("b200q_fake_quant_int", x.data_ptr(), y.data_ptr(), _dt(x), x.numel(), amax.data_ptr(), _dt(amax),
         amax.numel(), int(outer), int(num_bits), int(bool(unsigned)), int(bool(narrow_range)), _stream(x))
    return y


def fake_quant_fp8(x, amax=None, outer=1, out=None, eager=False):
    """FP8-E4M3 fake quant (amax=None: plain torch-style cast round trip).  ``eager``: the scale rule of the
    reference's _fp8_eager (reciprocal * 448) instead of the CUDA extension's 448 / amax."""
    x = _prep(x, "x")
    y = _out_arg(out, x)
    if amax is None:
        call("b200q_fake_quant_fp8", x.data_ptr(), y.data_ptr(), _dt(x), x.numel(), None, 0, 1, 1, _stream(x))
        return y
    amax = _amax_arg(amax, x)
    call("b200q_fake_quant_fp8_eager" if eager else "b200q_fake_quant_fp8", x.data_ptr(), y.data_ptr(), _dt(x),
         x.numel(), amax.data_ptr(), _dt(amax), amax.numel(), int(outer), _stream(x))
    return y


def fake_quant_nvfp4(x, global_amax, out=None):
    """NVFP4 dynamic block-16 fake quant along the last dim."""
    x = _prep(x, "x")
    global_amax = _amax_arg(global_amax, x)
    y = _out_arg(out, x)
    row_len = x.shape[-1] if x.dim() > 0 else 1
    n_rows = x.numel() // row_len if row_len else 0
    call("b200q_fake_quant_nvfp4", x.data_ptr(), y.data_ptr(), _dt(x), n_rows, row_len,
         global_amax.data_ptr(), _dt(global_amax), _stream(x))
    return y


HADAMARD_MAX_BLOCK = 32768


def _hadamard_shape(x, block_size):
    bs = int(block_size)
    if bs < 1 or bs & (bs - 1) or bs > HADAMARD_MAX_BLOCK:
        raise ValueError(f"Hadamard block_size must be a power of 2 no larger than {HADAMARD_MAX_BLOCK}, got {block_size}")
    row_len = x.shape[-1] if x.dim() > 0 else 1
    if row_len % bs:
        raise ValueError(f"the last dim {row_len} is not a multiple of the Hadamard block_size {bs}")
    return bs, row_len, (x.numel() // row_len if row_len else 0)


def hadamard(x, block_size, amax_slot=None):
    """Normalized Walsh-Hadamard transform of every contiguous block of ``block_size`` (a power of 2 up to 32768)
    elements along the last dim: fp32 butterflies in ascending stage order, one multiply by fl32(block_size ** -0.5),
    one rounding to x's dtype.  Returns a new tensor.  ``amax_slot`` (fp32 [1]): also folds max|y| into it, exactly as
    ``amax_per_tensor_(amax_slot, y)`` would."""
    bs, row_len, n_rows = _hadamard_shape(x, block_size)
    x = _prep(x, "x")
    if amax_slot is not None:
        _slots(amax_slot, "amax_slot")
    y = torch.empty_like(x)
    call("b200q_hadamard", x.data_ptr(), y.data_ptr(), _dt(x), n_rows, row_len, bs,
         None if amax_slot is None else amax_slot.data_ptr(), _stream(x))
    return y


def fake_quant_nvfp4_rotated(x, block_size, global_amax, rotate_back=False):
    """``fake_quant_nvfp4(hadamard(x, block_size), global_amax)``, rotated back with ``hadamard`` when
    ``rotate_back``: one pass, the same bits.  The last dim must be a multiple of 16 and of ``block_size``."""
    bs, row_len, n_rows = _hadamard_shape(x, block_size)
    x = _prep(x, "x")
    if row_len % 16:
        raise ValueError(f"rotated NVFP4 fake quant: the last dim {row_len} is not a multiple of 16")
    global_amax = _amax_arg(global_amax, x)
    y = torch.empty_like(x)
    call("b200q_fake_quant_nvfp4_rotated", x.data_ptr(), y.data_ptr(), _dt(x), n_rows, row_len, bs, int(bool(rotate_back)),
         global_amax.data_ptr(), _dt(global_amax), _stream(x))
    return y


def fake_quant_nvfp4_static(x, block_amax, global_amax=None, quantize_block_scales=True,
                            fp8_max_norm=448.0, out=None):
    """NVFP4 static fake quant: ``block_amax.numel() == x.numel() // 16`` calibrated amaxes."""
    x = _prep(x, "x")
    block_amax = _slots(block_amax.float().contiguous() if block_amax.dtype != torch.float32 or not block_amax.is_contiguous() else block_amax, "block_amax")
    n_blocks = block_amax.numel()
    if n_blocks * 16 != x.numel():
        raise B200QuantError("x.numel() must equal 16 * block_amax.numel()")
    if global_amax is None and quantize_block_scales:
        global_amax = torch.zeros(1, dtype=torch.float32, device=x.device)
        amax_per_tensor_(global_amax, block_amax)
    gptr = None
    if global_amax is not None:
        global_amax = global_amax.to(device=x.device, dtype=torch.float32).contiguous()
        gptr = global_amax.data_ptr()
    y = _out_arg(out, x)
    call("b200q_fake_quant_nvfp4_static", x.data_ptr(), y.data_ptr(), _dt(x), n_blocks, 16,
         block_amax.data_ptr(), gptr, int(bool(quantize_block_scales)), float(fp8_max_norm), _stream(x))
    return y


# ------------------------------------------------------------------------------------------------
# pack / unpack
# ------------------------------------------------------------------------------------------------
def pack_nvfp4(x, global_amax, block_amax=None, fp8_max_norm=448.0, block_size=16, wsf2=None):
    """-> (packed uint8 [..., K/2], scales float8_e4m3fn [..., K/block_size], wsf2 fp32 scalar).
    ``wsf2`` (instead of ``global_amax``): a caller-supplied weights_scaling_factor_2, used as is."""
    x = _prep(x, "x")
    k = x.shape[-1]
    n_rows = x.numel() // k
    packed = torch.empty((*x.shape[:-1], k // 2), dtype=torch.uint8, device=x.device)
    scales = torch.empty((*x.shape[:-1], k // block_size), dtype=torch.uint8, device=x.device)
    if wsf2 is not None:
        if block_amax is not None:
            raise B200QuantError("pack_nvfp4: wsf2 and block_amax are mutually exclusive")
        wsf2 = wsf2.to(device=x.device, dtype=torch.float32).reshape(()).contiguous()
        call("b200q_pack_nvfp4_scale2", x.data_ptr(), _dt(x), n_rows, k, int(block_size), wsf2.data_ptr(),
             packed.data_ptr(), scales.data_ptr(), _stream(x))
        return packed, scales.view(torch.float8_e4m3fn), wsf2
    global_amax = global_amax.to(device=x.device, dtype=torch.float32).contiguous()
    wsf2 = torch.empty((), dtype=torch.float32, device=x.device)
    if block_amax is None:
        call("b200q_pack_nvfp4", x.data_ptr(), _dt(x), n_rows, k, int(block_size), global_amax.data_ptr(), packed.data_ptr(),
             scales.data_ptr(), wsf2.data_ptr(), _stream(x))
    else:
        block_amax = block_amax.to(device=x.device, dtype=torch.float32).contiguous()
        call("b200q_pack_nvfp4_static", x.data_ptr(), _dt(x), n_rows, k, int(block_size), block_amax.data_ptr(),
             global_amax.data_ptr(), float(fp8_max_norm), packed.data_ptr(), scales.data_ptr(),
             wsf2.data_ptr(), _stream(x))
    return packed, scales.view(torch.float8_e4m3fn), wsf2


def unpack_nvfp4(packed, scales, wsf2, dtype=torch.bfloat16):
    packed = _prep(packed, "packed")
    scales = _prep(scales.view(torch.uint8), "scales")
    wsf2 = wsf2.to(device=packed.device, dtype=torch.float32).contiguous()
    k = packed.shape[-1] * 2
    n_rows = packed.numel() // packed.shape[-1]
    block_size = k // scales.shape[-1]               # the scale tensor's last dim tells the block size
    y = torch.empty((*packed.shape[:-1], k), dtype=dtype, device=packed.device)
    call("b200q_unpack_nvfp4", packed.data_ptr(), scales.data_ptr(), wsf2.data_ptr(), y.data_ptr(), _DT[dtype],
         n_rows, k, block_size, _stream(packed))
    return y


def pack_int4_blockwise(x, block_size):
    """INT4QTensor.quantize CUDA semantics -> (packed uint8 [numel/2], scales [n_blocks, 1] in x.dtype)."""
    x = _prep(x, "x")
    n = x.numel()
    scales = torch.empty((n // block_size, 1), dtype=x.dtype, device=x.device)
    packed = torch.empty(n // 2, dtype=torch.uint8, device=x.device)
    call("b200q_pack_int4_blockwise", x.data_ptr(), _dt(x), n, int(block_size), scales.data_ptr(),
         packed.data_ptr(), _stream(x))
    return packed, scales


def unpack_int4_blockwise(packed, scales, block_size):
    packed = _prep(packed, "packed")
    scales = _prep(scales, "scales")
    n = packed.numel() * 2
    y = torch.empty(n, dtype=scales.dtype, device=packed.device)
    call("b200q_unpack_int4_blockwise", packed.data_ptr(), scales.data_ptr(), _dt(scales), n, int(block_size),
         y.data_ptr(), _stream(packed))
    return y


def pack_int4_export(w, scale):
    """pack_int4_in_uint8: w [out, in], scale [out, in/block] -> uint8 [out/2, in]."""
    w = _prep(w, "w")
    scale = _prep(scale, "scale")
    out_dim, in_dim = w.shape[-2], w.shape[-1]
    block = in_dim // scale.shape[-1]
    packed = torch.empty((*w.shape[:-2], out_dim // 2, in_dim), dtype=torch.uint8, device=w.device)
    lead = w.numel() // (out_dim * in_dim)
    for i in range(lead):  # MoE [E, out, in]: one launch per expert
        wi = w.reshape(lead, out_dim, in_dim)[i]
        si = scale.reshape(lead, out_dim, -1)[i]
        pi = packed.reshape(lead, out_dim // 2, in_dim)[i]
        call("b200q_pack_int4_export", wi.data_ptr(), _dt(w), out_dim, in_dim, si.data_ptr(), _dt(scale),
             int(block), pi.data_ptr(), _stream(w))
    return packed


def pack_fp8(x, scale, outer=1):
    """(x / scale).to(float8_e4m3fn) with torch's promotion rules; returns a float8 tensor."""
    x = _prep(x, "x")
    scale = _amax_arg(scale, x)
    if scale.dtype == torch.float32 and x.dtype != torch.float32 and scale.numel() == 1 and scale.dim() > 0:
        # a one-element fp32 tensor WITH dims promotes x / scale to float32 in torch (no rounding of the
        # quotient to x.dtype); the C-ABI reads "n_scale == 1" as a 0-dim scale, so present it as a
        # two-entry per-channel scale whose first entry covers the whole tensor
        scale = scale.reshape(1).repeat(2)
        outer = max(x.numel(), 1)
    q = torch.empty(x.shape, dtype=torch.uint8, device=x.device)
    call("b200q_pack_fp8", x.data_ptr(), _dt(x), x.numel(), scale.data_ptr(), _dt(scale), scale.numel(),
         int(outer), q.data_ptr(), _stream(x))
    return q.view(torch.float8_e4m3fn)


def unpack_fp8(q, scale, dtype, outer=1):
    q = _prep(q.view(torch.uint8), "q")
    scale = _amax_arg(scale, q)
    y = torch.empty(q.shape, dtype=dtype, device=q.device)
    call("b200q_unpack_fp8", q.data_ptr(), scale.data_ptr(), _dt(scale), scale.numel(), int(outer),
         y.data_ptr(), _DT[dtype], q.numel(), _stream(q))
    return y


def pack_int8(x, scale, outer=1):
    """(x / scale).round().clamp(-128, 127).to(int8) with torch's promotion rules (INT8QTensor.quantize)."""
    x = _prep(x, "x")
    scale = _amax_arg(scale, x)
    if scale.dtype == torch.float32 and x.dtype != torch.float32 and scale.numel() == 1 and scale.dim() > 0:
        scale = scale.reshape(1).repeat(2)                      # see pack_fp8
        outer = max(x.numel(), 1)
    q = torch.empty(x.shape, dtype=torch.int8, device=x.device)
    call("b200q_pack_int8", x.data_ptr(), _dt(x), x.numel(), scale.data_ptr(), _dt(scale), scale.numel(),
         int(outer), q.data_ptr(), _stream(x))
    return q


def unpack_int8(q, scale, dtype, outer=1):
    q = _prep(q.view(torch.int8), "q")
    scale = _amax_arg(scale, q)
    y = torch.empty(q.shape, dtype=dtype, device=q.device)
    call("b200q_unpack_int8", q.data_ptr(), scale.data_ptr(), _dt(scale), scale.numel(), int(outer),
         y.data_ptr(), _DT[dtype], q.numel(), _stream(q))
    return y


def pack_nf4(x, block_size, scales=None):
    """NF4_quantize: flat x (numel % block_size == 0) -> (uint8 [numel / 2], scales [numel / block_size, 1] in
    x.dtype).  With ``scales`` given they are used as is (the extension call); else block |x| max is computed."""
    x = _prep(x, "x").reshape(-1)
    n = x.numel()
    packed = torch.empty(n // 2, dtype=torch.uint8, device=x.device)
    if scales is None:
        sc = torch.empty((n // block_size, 1), dtype=x.dtype, device=x.device)
        call("b200q_pack_nf4", x.data_ptr(), _dt(x), n, int(block_size), None, sc.data_ptr(), packed.data_ptr(),
             _stream(x))
        return packed, sc
    sc = _prep(scales, "scales")
    if sc.dtype != x.dtype or sc.numel() != n // block_size:
        raise ValueError("scales must have the input dtype and one entry per block")
    call("b200q_pack_nf4", x.data_ptr(), _dt(x), n, int(block_size), sc.data_ptr(), None, packed.data_ptr(), _stream(x))
    return packed, sc


def unpack_nf4(packed, scales, block_size):
    """NF4_dequantize: always bfloat16, flat [2 * numel(packed)]."""
    packed = _prep(packed, "packed").reshape(-1)
    scales = _prep(scales, "scales")
    y = torch.empty(packed.numel() * 2, dtype=torch.bfloat16, device=packed.device)
    call("b200q_unpack_nf4", packed.data_ptr(), scales.data_ptr(), _dt(scales), packed.numel(), int(block_size),
         y.data_ptr(), _stream(packed))
    return y


# ------------------------------------------------------------------------------------------------
# MX formats (E8M0 block scales)
# ------------------------------------------------------------------------------------------------
MX_FORMATS = {"E4M3": 0, "E5M2": 1, "INT8": 2, "E0M3": 3, "E1M2": 4, "E3M0": 5, "E2M1": 6, "E3M2": 7, "E2M3": 8,
              "E8M0": 9}


def fake_quant_mx(x, block_size, elem_format, out=None):
    """fused_amax_convert(x, block_size, elem_format, E8M0): blocks along the last dim."""
    x = _prep(x, "x")
    fmt = MX_FORMATS[elem_format] if isinstance(elem_format, str) else int(elem_format)
    y = _out_arg(out, x)
    k = x.shape[-1] if x.dim() else 1
    call("b200q_fake_quant_mx", x.data_ptr(), y.data_ptr(), _dt(x), x.numel() // max(k, 1), k, int(block_size), fmt,
         _stream(x))
    return y


def pack_mxfp8(x, scale=None):
    """MXFP8QTensor.quantize[_with_scale]: (float8_e4m3fn [..., K], uint8 scale [..., ceil(K / 32)])."""
    x = _prep(x, "x")
    k = x.shape[-1]
    rows = x.numel() // max(k, 1)
    q = torch.empty(x.shape, dtype=torch.uint8, device=x.device)
    if scale is None:
        s = torch.empty((*x.shape[:-1], (k + 31) // 32), dtype=torch.uint8, device=x.device)
        call("b200q_pack_mxfp8", x.data_ptr(), _dt(x), rows, k, None, q.data_ptr(), s.data_ptr(), _stream(x))
    else:
        s = _prep(scale, "scale")
        if s.dtype != torch.uint8 or s.numel() != rows * ((k + 31) // 32):
            raise ValueError("scale must be uint8 (E8M0) with one entry per 32-element block")
        call("b200q_pack_mxfp8", x.data_ptr(), _dt(x), rows, k, s.data_ptr(), q.data_ptr(), None, _stream(x))
    return q.view(torch.float8_e4m3fn), s


def unpack_mxfp8(q, scale, dtype):
    q = _prep(q.view(torch.uint8), "q")
    scale = _prep(scale, "scale")
    k = q.shape[-1]
    y = torch.empty(q.shape, dtype=dtype, device=q.device)
    call("b200q_unpack_mxfp8", q.data_ptr(), scale.data_ptr(), q.numel() // max(k, 1), k, y.data_ptr(), _DT[dtype],
         _stream(q))
    return y


def pack_mxfp4(x, block_size=32):
    """MXFP4QTensor.quantize: (uint8 [..., K / 2], uint8 scale [numel / block_size, 1])."""
    x = _prep(x, "x")
    if x.numel() % block_size or x.shape[-1] % 2:
        raise ValueError("numel must be a multiple of block_size and the last dim even")
    nb = x.numel() // block_size
    q = torch.empty((*x.shape[:-1], x.shape[-1] // 2), dtype=torch.uint8, device=x.device)
    s = torch.empty((nb, 1), dtype=torch.uint8, device=x.device)
    call("b200q_pack_mxfp4", x.data_ptr(), _dt(x), nb, int(block_size), q.data_ptr(), s.data_ptr(), _stream(x))
    return q, s


def unpack_mxfp4(q, scale, block_size, dtype):
    q = _prep(q, "q")
    scale = _prep(scale, "scale")
    nb = q.numel() * 2 // block_size
    y = torch.empty((*q.shape[:-1], q.shape[-1] * 2), dtype=dtype, device=q.device)
    call("b200q_unpack_mxfp4", q.data_ptr(), scale.data_ptr(), nb, int(block_size), y.data_ptr(), _DT[dtype],
         _stream(q))
    return y


def convert_to_exmy(x: float, elem_format) -> float:
    """Host scalar twin of cuda_ext_mx.convert_to_exmy."""
    from ._lib import load

    fmt = MX_FORMATS[elem_format] if isinstance(elem_format, str) else int(elem_format)
    return float(load().b200q_convert_to_exmy(float(x), fmt))


# ------------------------------------------------------------------------------------------------
# scale searches
# ------------------------------------------------------------------------------------------------
def scale_cols(x, scale, out=None):
    x = _prep(x, "x")
    scale = _amax_arg(scale, x)
    c = scale.numel()
    y = _out_arg(out, x)
    call("b200q_scale_cols", x.data_ptr(), y.data_ptr(), _dt(x), x.numel() // c, c, scale.data_ptr(),
         _dt(scale), _stream(x))
    return y


def awq_scale_fake_quant(w, col_scale, block_size, num_bits=4, narrow_range=False, out=None):
    w = _prep(w, "w")
    col_scale = _amax_arg(col_scale, w)
    c = w.shape[-1]
    y = _out_arg(out, w)
    call("b200q_awq_scale_fake_quant", w.data_ptr(), y.data_ptr(), _dt(w), w.numel() // c, c,
         col_scale.data_ptr(), _dt(col_scale), int(block_size), int(num_bits), int(bool(narrow_range)), _stream(w))
    return y


def awq_weight_scale_sums_(sums, w, block_size):
    w = _prep(w, "w")
    _slots(sums, "sums")
    c = w.shape[-1]
    call("b200q_awq_weight_scale_sums", w.data_ptr(), _dt(w), w.numel() // c, c, int(block_size),
         sums.data_ptr(), _stream(w))
    return sums


def mse_sweep_(loss, x, amax0, mult, num_bits=8, unsigned=False, narrow_range=False):
    """loss[k] += sum (fq(x; amax0*mult[k]) - x)^2, fp64; num_bits=0 selects FP8-E4M3."""
    x = _prep(x, "x")
    if loss.dtype != torch.float64 or not loss.is_cuda:
        raise B200QuantError("loss must be a float64 CUDA tensor")
    amax0 = amax0.to(device=x.device, dtype=torch.float32).contiguous()
    mult = mult.to(device=x.device, dtype=torch.float32).contiguous()
    call("b200q_mse_sweep", x.data_ptr(), _dt(x), x.numel(), amax0.data_ptr(), mult.data_ptr(), mult.numel(),
         int(num_bits), int(bool(unsigned)), int(bool(narrow_range)), loss.data_ptr(), _stream(x))
    return loss


def mse_sweep_rows_(loss, x, amax0, mult, num_bits=8, unsigned=False, narrow_range=False, cand_dtype=None,
                    round_mult=True):
    """Per-row MSE sweep: x viewed as [R, L] with R = amax0.numel(); loss [n_cand, R] fp32 +=
    sum_j (fq(x[r, j]; round_A(amax0[r] * m_k)) - x[r, j])^2, A = cand_dtype (default: amax0.dtype),
    m_k = round_A(mult[k]) (torch's CUDA rule, default) or mult[k] (torch's CPU rule, round_mult=False)."""
    x = _prep(x, "x")
    r = amax0.numel()
    if r == 0 or x.numel() % r:
        raise B200QuantError("x.numel() must be a multiple of amax0.numel()")
    cand_dtype = cand_dtype or amax0.dtype
    if loss.dtype != torch.float32 or not loss.is_cuda or not loss.is_contiguous() or loss.numel() != mult.numel() * r:
        raise B200QuantError("loss must be a contiguous float32 CUDA tensor of n_cand * n_rows elements")
    a0 = amax0.to(device=x.device, dtype=torch.float32).contiguous()
    mult = mult.to(device=x.device, dtype=torch.float32).contiguous()
    call("b200q_mse_sweep_rows", x.data_ptr(), _dt(x), r, x.numel() // r, a0.data_ptr(), mult.data_ptr(),
         mult.numel(), _DT[cand_dtype], int(bool(round_mult)), int(num_bits), int(bool(unsigned)),
         int(bool(narrow_range)), loss.data_ptr(), _stream(x))
    return loss


_FP8_CAND_CACHE: dict = {}


def fp8_scale_candidates(device) -> torch.Tensor:
    """The 126 positive finite E4M3 values / 448 as TORCH evaluates them on ``device``
    (kernels/quantization/gemm/_fp8_scale_candidates.py:28-33): on CUDA ``/ 448.0`` is a multiply by fl(1 / 448)."""
    device = torch.device(device)
    c = _FP8_CAND_CACHE.get(device)
    if c is None:
        v = torch.arange(0, 128, dtype=torch.uint8, device=device).view(torch.float8_e4m3fn).float()
        c = (v[torch.isfinite(v) & (v > 0)] / 448.0).contiguous()
        _FP8_CAND_CACHE[device] = c
    return c


def nvfp4_fp8_scale_sweep(w, global_amax, candidates="device", hessian=None):
    """Per-16-block argmin over the FP8-E4M3 block-scale candidates (``nvfp4_fp8_scale_sweep[_hessian]``,
    kernels/quantization/gemm/nvfp4_fp8_sweep.py:127-290) -> fp32 ``best_amax`` [n_blocks].

    ``candidates``: "device" (default) = the candidate set as torch builds it on the weight's device, i.e. what a GPU
    run of the reference sweeps; "ieee" = e4m3 / 448 by IEEE division (what torch builds on CPU -- the committed
    fixtures); or a tensor.  ``hessian`` ([cin / 16, 16, 16] fp32): minimise dw^T H dw instead of the squared error."""
    w = _prep(w, "w")
    global_amax = global_amax.detach().to(device=w.device, dtype=torch.float32).contiguous()
    n_blocks = w.numel() // 16
    best = torch.empty(n_blocks, dtype=torch.float32, device=w.device)
    if isinstance(candidates, str):
        cand = None if candidates == "ieee" else fp8_scale_candidates(w.device)
    else:
        cand = candidates.to(device=w.device, dtype=torch.float32).contiguous()
    if hessian is None:
        call("b200q_nvfp4_fp8_scale_sweep_ex", w.data_ptr(), _dt(w), n_blocks, global_amax.data_ptr(),
             None if cand is None else cand.data_ptr(), 126 if cand is None else cand.numel(), best.data_ptr(), _stream(w))
        return best
    if hessian.dim() != 3 or hessian.shape[1] != 16 or hessian.shape[2] != 16:
        raise B200QuantError(f"hessian must have shape [n_cin_blocks, 16, 16], got {tuple(hessian.shape)}")
    n_cin = hessian.shape[0]
    if n_blocks % n_cin:
        raise B200QuantError(f"n_blocks ({n_blocks}) is not divisible by n_cin_blocks ({n_cin})")
    if cand is None:
        cand = fp8_scale_candidates("cpu").to(w.device)
    cand_scales, cand_amaxes = hessian_sweep_candidates(global_amax, cand)
    h = hessian.detach().to(device=w.device, dtype=torch.float32).contiguous()
    call("b200q_nvfp4_fp8_scale_sweep_hessian", w.data_ptr(), _dt(w), n_blocks // n_cin, n_cin, cand_scales.data_ptr(),
         cand_amaxes.data_ptr(), cand.numel(), h.data_ptr(), best.data_ptr(), _stream(w))
    return best


def hessian_sweep_candidates(global_amax, cand):
    """``(cand_scales, cand_amaxes)`` of the Hessian-weighted sweep (nvfp4_fp8_sweep.py:272-275), fp32 on ``cand``'s
    device: ``cand_amaxes = cand * g`` and ``cand_scales = compute_fp4_scales(cand_amaxes, g, True)`` (fp4_kernel.py:
    217-251), i.e. ``cand_amaxes / 6`` through the FP8 fake quant at amax ``g / 6``."""
    g = global_amax.detach().to(device=cand.device, dtype=torch.float32).reshape(())
    cand_amaxes = (cand * g).contiguous()
    cand_scales = fake_quant_fp8((cand_amaxes / 6.0).contiguous(), (g * (448.0 / 448.0) / 6.0).reshape(1))
    return cand_scales, cand_amaxes


def nvfp4_static_mse_sweep(w, amax0, global_amax, mult, fp8_max_norm=448.0, loss_out=None):
    """Static NVFP4 per-block multiplier search (``MseCalibrator`` on the blocked weight, calib/mse.py:84-172) ->
    fp32 ``best_amax`` [n_blocks] = ``amax0 * mult[argmin_k loss[k]]``, one launch.  ``w``: the weight, 16 elements
    per block (bf16, fp16 or fp32); ``amax0``: the fp32 per-block amax; ``mult``: at most 128 fp32 multipliers
    (``torch.linspace(start, stop, steps)`` on the weight's device, as the calibrator builds them); ``fp8_max_norm``:
    256 for Four-Over-Six, else 448.  ``loss_out``: an optional fp32 [n_cand, n_blocks] tensor that receives
    every block's loss per candidate."""
    w = _prep(w, "w")
    n_blocks = w.numel() // 16
    if n_blocks * 16 != w.numel():
        raise B200QuantError("w.numel() must be a multiple of 16")
    if amax0.numel() != n_blocks:
        raise B200QuantError(f"amax0 has {amax0.numel()} values for {n_blocks} blocks")
    a0 = amax0.detach().to(device=w.device, dtype=torch.float32).contiguous()
    g = global_amax.detach().to(device=w.device, dtype=torch.float32).reshape(-1).contiguous()
    if g.numel() != 1:
        raise B200QuantError("global_amax must hold one value")
    mult = mult.detach().to(device=w.device, dtype=torch.float32).contiguous()
    if loss_out is not None and (loss_out.dtype != torch.float32 or not loss_out.is_cuda
                                 or not loss_out.is_contiguous() or loss_out.numel() != mult.numel() * n_blocks):
        raise B200QuantError("loss_out must be a contiguous float32 CUDA tensor of n_cand * n_blocks elements")
    best = torch.empty(n_blocks, dtype=torch.float32, device=w.device)
    call("b200q_nvfp4_static_mse_sweep", w.data_ptr(), _dt(w), n_blocks, a0.data_ptr(), g.data_ptr(),
         mult.data_ptr(), mult.numel(), float(fp8_max_norm), best.data_ptr(),
         None if loss_out is None else loss_out.data_ptr(), _stream(w))
    return best


# ------------------------------------------------------------------------------------------------
# GPTQ weight calibration
# ------------------------------------------------------------------------------------------------
GPTQ_INT, GPTQ_FP8, GPTQ_NVFP4_STATIC, GPTQ_NVFP4_DYNAMIC = 0, 1, 2, 3
GPTQ_PER_TENSOR_COL_BLOCK = 1 << 62      # an amax column block wider than any matrix: one amax per row / tensor


def _rows_view(t: torch.Tensor, name: str) -> torch.Tensor:
    if not t.is_cuda or t.dtype != torch.float32 or t.dim() != 2 or t.stride(1) != 1:
        raise B200QuantError(f"{name} must be a 2-D float32 CUDA tensor with unit column stride")
    return t


def gptq_block_update(w, u, fmt, amax, amax_row_stride=0, amax_col_block=GPTQ_PER_TENSOR_COL_BLOCK, col0=0,
                      num_bits=8, unsigned=False, narrow_range=False, global_amax=None):
    """The column loop of one GPTQ block (``b200q_gptq_block``): ``w`` [rows, nb] fp32 (a column slice of the working
    matrix, row stride free) is replaced in place by its fake-quantized columns; ``u`` [nb, nb] fp32 is the block of
    the upper Cholesky factor of the inverse Hessian (any strides: a column-major block is copied, nb x nb floats).
    Returns the scaled errors E [rows, nb] (fp32)."""
    _rows_view(w, "w")
    if u.is_cuda and u.dtype == torch.float32 and u.dim() == 2 and u.stride(1) != 1:
        u = u.contiguous()           # the factor of torch.linalg.cholesky(upper=True) is column-major
    _rows_view(u, "u")
    rows, nb = w.shape
    if u.shape[0] < nb or u.shape[1] < nb:
        raise B200QuantError(f"u {tuple(u.shape)} is smaller than the block ({nb} columns)")
    amax = _prep(amax, "amax")
    _dt(amax)
    g = None
    if global_amax is not None:
        g = _prep(global_amax.reshape(-1), "global_amax")
        if g.dtype != torch.float32:
            raise B200QuantError("global_amax must be float32")
    e = torch.empty(rows, nb, dtype=torch.float32, device=w.device)
    call("b200q_gptq_block", w.data_ptr(), w.stride(0), rows, nb, u.data_ptr(), u.stride(0), e.data_ptr(), int(fmt),
         amax.data_ptr(), _dt(amax), int(amax_row_stride), int(amax_col_block), int(col0), int(num_bits),
         int(bool(unsigned)), int(bool(narrow_range)), None if g is None else g.data_ptr(), _stream(w))
    return e


def gptq_quantizer_desc(quantizer, shape, block_size=None, device=None) -> dict | None:
    """The ``gptq_block_update`` description of a calibrated weight quantizer for a [out, in] weight, or None when
    its fake quant is outside the kernel's scope (MX, 2-D blocks, NF4, pre_quant_scale, rotation, bias, padded block
    layouts, NVFP4 blocks straddling GPTQ blocks of ``block_size`` columns, calibrated state on another device than
    ``device``, or no calibrated ``_amax``: a dynamic per-tensor amax is taken over the whole working matrix at every
    column).  Reads attributes that the engine's and the reference's quantizers share."""
    desc = _gptq_quantizer_desc(quantizer, shape)
    if desc is None:
        return None
    if block_size is not None and desc["fmt"] in (GPTQ_NVFP4_STATIC, GPTQ_NVFP4_DYNAMIC) and block_size % 16:
        return None
    if device is not None and any(isinstance(t, torch.Tensor) and t.device != torch.device(device)
                                  for t in (desc["amax"], desc.get("global_amax"))):
        return None
    return desc


def _gptq_quantizer_desc(quantizer, shape):
    out_f, in_f = int(shape[0]), int(shape[1])
    q = quantizer
    if getattr(q, "_disabled", False) or not getattr(q, "_fake_quant", True) or getattr(q, "_lsq", False):
        return None
    if getattr(q, "pre_quant_scale", None) is not None or getattr(q, "rotate_is_enabled", False) \
            or getattr(q, "bias", None) or getattr(q, "is_mx_format", False):
        return None
    amax = getattr(q, "_amax", None)
    if not isinstance(amax, torch.Tensor) or not amax.is_cuda or amax.dtype not in _DT:
        return None
    nbits = q._num_bits
    bs = q._block_sizes
    if bs:
        keys = [k for k in bs if isinstance(k, int)]
        if len(keys) != 1 or keys[0] not in (-1, 1) or bs[keys[0]] is None or bs.get("four_over_six", False) \
                or bs.get("scale_block_sizes"):
            return None
        cb = int(bs[keys[0]])
        if in_f % cb:
            return None
        scale_bits = bs.get("scale_bits")
        if bs.get("type", "static") == "dynamic":
            if nbits == (2, 1) and scale_bits == (4, 3) and cb == 16 and amax.numel() == 1:
                return {"fmt": GPTQ_NVFP4_DYNAMIC, "amax": amax}
            return None
        if nbits == (2, 1):
            g = getattr(q, "_global_amax", None)
            if scale_bits == (4, 3) and cb == 16 and isinstance(g, torch.Tensor) and g.numel() == 1 \
                    and amax.numel() == out_f * in_f // 16:
                return {"fmt": GPTQ_NVFP4_STATIC, "amax": amax.float(), "amax_row_stride": in_f // 16,
                        "amax_col_block": 16, "global_amax": g.float()}
            return None
        if scale_bits is not None or (isinstance(nbits, tuple) and nbits != (4, 3)) \
                or amax.numel() != out_f * in_f // cb:
            return None
        desc = {"amax": amax, "amax_row_stride": in_f // cb, "amax_col_block": cb}
    elif isinstance(nbits, tuple) and nbits != (4, 3):
        return None
    elif amax.numel() == 1:
        desc = {"amax": amax}
    elif amax.dim() == 2 and tuple(amax.shape) == (out_f, 1):
        desc = {"amax": amax, "amax_row_stride": 1}
    else:
        return None
    if nbits == (4, 3):
        desc["fmt"] = GPTQ_FP8
    else:
        desc.update(fmt=GPTQ_INT, num_bits=nbits, unsigned=q._unsigned, narrow_range=q._narrow_range)
    return desc


def gptq_blockwise_update(weight, h_inv, block_size, quantizer, desc=None):
    """``gptq_blockwise_update`` (utils/calib_utils.py:241-276) with the column loop of every block in one kernel:
    ``weight`` [out, in] fp32 is updated in place; per block, ``gptq_block_update`` then the reference's trailing
    ``weight[:, be:].addmm_(E, h_inv[bs:be, be:], alpha=-1)`` (a cuBLAS GEMM through torch).  Raises for a quantizer
    outside the kernel's scope (``gptq_quantizer_desc`` is None); callers take the composed loop there."""
    if desc is None:
        desc = gptq_quantizer_desc(quantizer, weight.shape, block_size, weight.device)
    if desc is None:
        raise B200QuantError("gptq_blockwise_update: the weight quantizer is outside the GPTQ kernel's scope")
    if desc["fmt"] in (GPTQ_NVFP4_STATIC, GPTQ_NVFP4_DYNAMIC) and block_size % 16:
        raise B200QuantError(f"gptq_blockwise_update: NVFP4 blocks straddle GPTQ blocks of {block_size} columns")
    _rows_view(weight, "weight")
    if not h_inv.is_cuda or h_inv.dtype != torch.float32 or h_inv.dim() != 2:
        raise B200QuantError("h_inv must be a 2-D float32 CUDA tensor")
    num_cols = weight.shape[1]
    for bs in range(0, num_cols, block_size):
        be = min(bs + block_size, num_cols)
        errs = gptq_block_update(weight[:, bs:be], h_inv[bs:be, bs:be], col0=bs, **desc)
        weight[:, be:].addmm_(errs, h_inv[bs:be, be:], alpha=-1)
    return weight


def selftest_fastdiv(seed: int, n: int) -> int:
    import ctypes

    m = ctypes.c_ulonglong(0)
    call("b200q_selftest_fastdiv", int(seed), int(n), ctypes.byref(m))
    return int(m.value)


def selftest_e2m1_round() -> int:
    import ctypes

    m = ctypes.c_ulonglong(0)
    call("b200q_selftest_e2m1_round", ctypes.byref(m))
    return int(m.value)


def _on_tensor_device(fn):
    """The C-ABI launches on the calling thread's current device.  Every public op runs with the device of its
    first CUDA tensor argument current and restores the previous one afterwards (nothing is cached: torch's
    current device can change between calls)."""

    @functools.wraps(fn)
    def wrapper(*args, **kwargs):
        for a in args:
            if isinstance(a, torch.Tensor) and a.is_cuda:
                if a.device.index != torch.cuda.current_device():
                    with torch.cuda.device(a.device):
                        return fn(*args, **kwargs)
                break
        return fn(*args, **kwargs)

    return wrapper


for _n, _f in list(globals().items()):
    if callable(_f) and not isinstance(_f, type) and getattr(_f, "__module__", None) == __name__ \
            and not _n.startswith("_") \
            and _n not in ("selftest_fastdiv", "selftest_e2m1_round", "convert_to_exmy"):
        globals()[_n] = _on_tensor_device(_f)

__all__ = [n for n in dir() if not n.startswith("_") and n not in ("torch", "functools", "annotations")]

"""ops.live_block_ranges: which blocks of each output the fix-up of the fused collect + fake quant redoes or rewrites,
and which buffer layouts it refuses.  Pure host arithmetic on (address, bytes) pairs."""

import pytest

from model_optimizer_b200.engine import LLAMA3_8B
from model_optimizer_b200.ops import B200QuantError, live_block_ranges

BLK = 32   # one 16-element bf16 block


def _writers(outputs):
    """Every entry writes its output in order: {(buffer base, block): [entries writing it, in order]}."""
    w = {}
    for i, (a, n) in enumerate(outputs):
        for b in range(n // BLK):
            w.setdefault((a, b), []).append(i)
    return w


def test_ring_of_four_like_the_engine():
    tokens = 8
    cins = [cin for _, cin, _ in LLAMA3_8B.linears()] * 3           # 21 entries, widths 4096 / 14336 mixed
    nbytes = [tokens * c * 2 for c in cins]
    ring = [1 << (40 + k) for k in range(4)]                          # 4 buffers, far apart
    inputs, a = [], 1 << 30
    for n in nbytes:
        inputs.append((a, n))
        a += n
    outputs = [(ring[i % 4], n) for i, n in enumerate(nbytes)]
    ranges = live_block_ranges(inputs, outputs, BLK)
    writers = _writers(outputs)
    # each written block of each buffer lies in exactly one entry's live range: that of the entry that writes it last;
    # it is contested exactly when an earlier entry writes it too
    owner = {}
    for i, ((base, n), (lf, ct)) in enumerate(zip(outputs, ranges)):
        assert 0 <= lf <= ct <= n // BLK
        for b in range(lf, n // BLK):
            assert (base, b) not in owner
            owner[(base, b)] = i
            assert (b < ct) == (len(writers[(base, b)]) > 1)
    assert owner == {k: v[-1] for k, v in writers.items()}
    assert [lf for lf, _ in ranges[-4:]] == [0, 0, 0, 0]              # nothing comes after the last four
    assert [ct for _, ct in ranges[:4]] == [lf for lf, _ in ranges[:4]]   # nothing comes before the first four


def test_distinct_outputs_are_all_live_and_uncontested():
    inputs = [(1000 + 64 * i, 64) for i in range(5)]
    outputs = [(10_000 + 128 * i, 64) for i in range(5)]
    assert live_block_ranges(inputs, outputs, BLK) == [(0, 0)] * 5


def test_output_overlapping_an_input_is_refused():
    inputs = [(0, 4096), (8192, 4096)]
    with pytest.raises(B200QuantError, match="overlaps an input"):
        live_block_ranges(inputs, [(1 << 20, 4096), (8192 + 1024, 64)], BLK)
    with pytest.raises(B200QuantError, match="overlaps an input"):
        live_block_ranges(inputs, [(0, 4096), (1 << 20, 64)], BLK)       # in place
    # touching without overlap is fine
    assert live_block_ranges(inputs, [(4096, 4096), (12288, 64)], BLK) == [(0, 0), (0, 0)]


def test_outputs_overlapping_at_different_bases_are_refused():
    inputs = [(0, 256), (256, 256)]
    with pytest.raises(B200QuantError, match="without sharing a base"):
        live_block_ranges(inputs, [(1 << 20, 256), ((1 << 20) + 64, 256)], BLK)
    # same base: the later output covers a prefix of the earlier one
    assert live_block_ranges(inputs, [(1 << 20, 256), (1 << 20, 64)], BLK) == [(2, 2), (0, 2)]
    # a later, LONGER output at the same base hides the earlier one completely
    assert live_block_ranges(inputs, [(1 << 20, 64), (1 << 20, 256)], BLK) == [(2, 2), (0, 2)]

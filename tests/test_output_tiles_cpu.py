"""ops.output_tiles: the per-tile store-order bookkeeping of the fused collect + fake quant, against a brute-force replay
of every entry's block writes in table order.  Pure host arithmetic on (address, bytes) pairs."""

import random

import pytest

from model_optimizer_b200.engine import LLAMA3_8B, TINY
from model_optimizer_b200.ops import output_tiles, second_pass_tiles


def _replay(outputs, block_bytes, tile_blocks):
    """Write every entry's blocks in order; per (buffer, tile): (writers in order, {block: last writer})."""
    tiles = {}
    for i, (a, n) in enumerate(outputs):
        for b in range(n // block_bytes):
            w, last = tiles.setdefault((a, b // tile_blocks), ([], {}))
            if not w or w[-1] != i:
                w.append(i)
            last[b] = i
    return tiles


def _check(outputs, block_bytes, tile_blocks):
    tile0, owner, expected, preflag, pieces = output_tiles(outputs, block_bytes, tile_blocks)
    tiles = _replay(outputs, block_bytes, tile_blocks)
    # entries sharing a buffer share their tile numbering; different buffers get disjoint tile ranges
    index = {}
    for i, (a, _) in enumerate(outputs):
        assert tile0[i] == tile0[[j for j, (b, _) in enumerate(outputs) if b == a][0]]
    for (a, k), _ in tiles.items():
        i = [j for j, (b, _) in enumerate(outputs) if b == a][0]
        index[(a, k)] = tile0[i] + k
    assert len(set(index.values())) == len(index) == len(owner)
    want_pieces = set()
    for key, (writers, last) in tiles.items():
        t = index[key]
        assert owner[t] == writers[-1]
        assert expected[t] == len(writers) - 1
        live_entries = sorted(set(last.values()))
        assert preflag[t] == (len(live_entries) > 1)
        if preflag[t]:
            for e in live_entries:
                blocks = sorted(b for b, w in last.items() if w == e)
                assert blocks == list(range(blocks[0], blocks[-1] + 1))
                want_pieces.add((e, blocks[0], blocks[-1] + 1))
    assert sorted(pieces) == sorted(want_pieces)
    assert len(pieces) == len(want_pieces)
    # the second pass: exactly the tiles an entry writes last while an earlier entry writes them too
    second = second_pass_tiles(outputs, block_bytes, tile_blocks)
    want_second = {(ws[-1], k) for (a, k), (ws, _) in tiles.items() if len(ws) > 1}
    got_second = {(i, k) for i, (k0, k1) in enumerate(second) for k in range(k0, k1)}
    assert got_second == want_second


@pytest.mark.parametrize("block_bytes", [64, 32], ids=["fp32", "16bit"])
@pytest.mark.parametrize("ring", [1, 2, 3, 4, 5])
def test_random_tables_against_replay(ring, block_bytes):
    rng = random.Random(1000 * ring + block_bytes)
    tile_blocks = 8
    for _ in range(40):
        bases = [(1 << 40) + (k << 30) for k in range(ring)]
        n_entries = rng.randint(1, 14)
        outputs = []
        for i in range(n_entries):
            kind = rng.random()
            if kind < 0.3:
                nblk = tile_blocks * rng.randint(1, 6)                       # live bounds on tile edges
            elif kind < 0.4:
                nblk = 0
            else:
                nblk = rng.randint(1, 6 * tile_blocks)                       # and inside tiles
            base = bases[i % ring] if rng.random() < 0.8 else (1 << 50) + (i << 30)   # some outputs of their own
            outputs.append((base, nblk * block_bytes))
        _check(outputs, block_bytes, tile_blocks)


def test_engine_layout_at_512_block_tiles():
    # TINY at 40 tokens: entries of 640 and 1280 blocks in a ring of 4, so live bounds fall inside tile 1
    cins = [cin for _, cin, _ in TINY.linears()] * TINY.n_layers
    outputs = [((1 << 40) + ((i % 4) << 30), 40 * c * 2) for i, c in enumerate(cins)]
    _check(outputs, 32, 512)
    _, _, _, preflag, pieces = output_tiles(outputs, 32)
    assert any(preflag) and pieces


def test_bench_table_has_nothing_to_rewrite():
    # bench.py's step: 224 activations [4096, cin] into a ring of 4 buffers; every live bound is tile-aligned
    cins = [cin for _, cin, _ in LLAMA3_8B.linears()] * LLAMA3_8B.n_layers
    outputs = [((1 << 40) + ((i % 4) << 36), 4096 * c * 2) for i, c in enumerate(cins)]
    tile0, owner, expected, preflag, pieces = output_tiles(outputs, 32)
    assert len(owner) == 4 * 4096 * 14336 // 16 // 512
    assert not any(preflag) and pieces == []
    assert all(e >= 0 for e in expected) and sorted(set(tile0)) == [0, 7168, 2 * 7168, 3 * 7168]

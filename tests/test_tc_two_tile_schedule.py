"""Host logic of the merged-launch schedule (csrc/conv_tc.cu:tc_schedule) with two-tile units and the automatic split into
one-tile items when the two-tile units are too coarse for the SMs.  No GPU needed."""
from tests.test_native_abi import _schedule


def _covers_every_tile_once(items, n_layers, B, tiles, col_blocks):
    got = sorted((int(l), int(nb), int(b), int(t0) // 128 + k)
                 for l, nb, b, t0, mt in items for k in range(int(mt)))
    want = sorted((l, nb, b, t) for l in range(n_layers) for nb in range(col_blocks) for b in range(B) for t in range(tiles))
    return got == want


def test_coarse_two_tile_units_are_split_until_balanced():
    """Stage 0 shape (C = 256, 2 column blocks, k 3 / 7 / 11) at 4 clips x 1024 rows: 96 two-tile units on 132 CTAs
    leave CTAs idle; split into one-tile items they balance above 0.95."""
    items, off, bal = _schedule([3, 7, 11], [0, 0, 0], [0, 0, 0], 4, 1024, 2, 2, False, Cin=256)
    assert _covers_every_tile_once(items, 3, 4, 8, 2)
    assert (items[:, 4] == 1).all() and bal >= 0.95
    assert off[0] == 0 and off[-1] == len(items) and (off[1:] - off[:-1] <= 120).all()


def test_split_mixes_two_tile_and_one_tile_items():
    """Stage 2 shape (C = 64) at 4 clips x 41 tiles on 132 CTAs: 21 units per clip and layer, the last one tile, so
    one launch runs both kinds of items."""
    items, off, bal = _schedule([3, 7, 11], [0, 0, 0], [0, 0, 0], 4, 41 * 128, 2, 1, False, Cin=64)
    assert _covers_every_tile_once(items, 3, 4, 41, 1)
    assert set(items[:, 4].tolist()) == {1, 2}
    assert 0.8 < bal <= 1.0


def test_split_keeps_chain_order_and_odd_tile_tails():
    """Chain-ordered step (the ResBlock sum), 5 clips x 3 tiles on 8 CTAs: split units keep layers 0, 1, 2 of a tile back
    to back, and the one-tile tail of every clip stays one tile."""
    items, off, bal = _schedule([3, 7, 11], [1, 1, 1], [0, 1, 1], 5, 3 * 128 - 40, 2, 1, True, grid=8)
    assert _covers_every_tile_once(items, 3, 5, 3, 1)
    for c in range(len(off) - 1):
        mine = items[off[c]:off[c + 1]]
        for i in range(0, len(mine), 3):
            assert mine[i:i + 3, 0].tolist() == [0, 1, 2]
            assert (mine[i:i + 3, 1:] == mine[i, 1:]).all()
    assert not ((items[:, 3] == 256) & (items[:, 4] == 2)).any()
    assert 0 < bal <= 1.0

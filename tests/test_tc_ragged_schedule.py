"""Host logic of ragged batches in the wgmma conv planner (csrc/conv_tc.cu: tc_schedule with per-clip row bounds, through
svb_tc_ragged_schedule_probe): every live (clip, tile) is scheduled exactly once, no item starts at or past its clip's end, every
item carries its clip's bound, chain-ordered lists keep the layers of a unit together and in order, and equal lengths give the
items of the uniform probes.  No GPU needed."""
import ctypes

import numpy as np
import pytest

K_MAX_ITEMS = 120
GRID = 132
arr = lambda v: np.ascontiguousarray(v, dtype=np.int32)


def _lib():
    from neuralsvb_b200 import _native
    return _native


def ragged(KS, has_res, accum, lengths, MT=2, col_blocks=1, chain=False, KS2=None, Cin=64, grid=GRID):
    N = _lib()
    k, hr, ac, ln = arr(KS), arr(has_res), arr(accum), arr(lengths)
    k2 = None if KS2 is None else arr(KS2)
    cap = 400000
    items, off, P, bal = np.zeros((cap, 6), np.int32), np.zeros(grid + 1, np.int32), ctypes.c_int32(), ctypes.c_double()
    cnt = N.check(N.lib().svb_tc_ragged_schedule_probe(len(KS), k.ctypes.data, None if k2 is None else k2.ctypes.data, hr.ctypes.data,
                                                       ac.ctypes.data, Cin, len(lengths), ln.ctypes.data, MT, col_blocks, int(chain),
                                                       grid, items.ctypes.data, cap, off.ctypes.data, ctypes.byref(P),
                                                       ctypes.byref(bal)), 'tc_ragged_schedule_probe')
    return items[:cnt], off, P.value, bal.value


def uniform(KS, has_res, accum, B, Tq, MT=2, col_blocks=1, chain=False, Cin=64, grid=GRID):
    N = _lib()
    k, hr, ac = arr(KS), arr(has_res), arr(accum)
    cap = 400000
    items, off, bal = np.zeros((cap, 5), np.int32), np.zeros(grid + 1, np.int32), ctypes.c_double()
    cnt = N.check(N.lib().svb_tc_schedule_probe(len(KS), k.ctypes.data, hr.ctypes.data, ac.ctypes.data, Cin, B, Tq, MT, col_blocks,
                                                int(chain), grid, items.ctypes.data, cap, off.ctypes.data, ctypes.byref(bal)),
                  'tc_schedule_probe')
    return items[:cnt], off


def uniform_fused(KS1, dil1, KS2, accum, B, Tq, chain, Cin=32, grid=GRID):
    N = _lib()
    k1, d1, k2, ac = arr(KS1), arr(dil1), arr(KS2), arr(accum)
    cap = 400000
    items, off, P, bal = np.zeros((cap, 7), np.int32), np.zeros(grid + 1, np.int32), ctypes.c_int32(), ctypes.c_double()
    cnt = N.check(N.lib().svb_tc_fused_schedule_probe(len(KS1), k1.ctypes.data, d1.ctypes.data, k2.ctypes.data, ac.ctypes.data, Cin, B,
                                                      Tq, int(chain), grid, items.ctypes.data, cap, off.ctypes.data, ctypes.byref(P),
                                                      ctypes.byref(bal)), 'tc_fused_schedule_probe')
    return items[:cnt], off, P.value


def check(items, off, n_layers, lengths, col_blocks, rows_per_item, chain, fused):
    """Coverage, bounds and ordering of one ragged list; rows_per_item(item) = output rows the item owns."""
    B = len(lengths)
    assert off[0] == 0 and off[-1] == len(items) and (np.diff(off) >= 0).all()
    assert (np.diff(off) <= K_MAX_ITEMS).all()
    Tmax = max(lengths)
    cover = np.zeros((n_layers, col_blocks, B, Tmax + 512), np.int32)
    for l, nb, b, t0, mt, bound in items:
        assert bound == lengths[b], (b, bound, lengths[b])          # the item carries its clip's row bound
        assert 0 <= t0 < lengths[b], (b, t0, lengths[b])              # no item starts at or past its clip's end
        if fused:
            assert mt == 2 and nb == 0
        else:
            assert mt in (1, 2) and t0 % 128 == 0
            assert t0 + 128 * (mt - 1) < lengths[b]                   # not even the second tile of an item is dead
        cover[l, nb, b, t0:t0 + rows_per_item(mt)] += 1
    for b, L in enumerate(lengths):
        # every live row of every (layer, column block, clip) exactly once
        assert (cover[:, :, b, :L] == 1).all(), b
        # tiles are whole: nothing is scheduled after the clip's last live tile
        if not fused:
            assert (cover[:, :, b, (L + 127) // 128 * 128:] == 0).all(), b
    if chain and n_layers > 1:
        for c in range(len(off) - 1):
            mine = items[off[c]:off[c + 1]]
            assert len(mine) % n_layers == 0
            for u in range(0, len(mine), n_layers):
                grp = mine[u:u + n_layers]
                assert list(grp[:, 0]) == list(range(n_layers))       # chain order: layers 0, 1, ... of one unit back to back
                assert (grp[:, 1:5] == grp[0, 1:5]).all()


LENGTHS = {
    'equal': [300] * 6,
    'one_frame_clip': [1, 517, 256, 33],
    'around_128k': [127, 128, 129, 255, 256, 257, 383, 384, 385],
    'around_P': [245, 246, 247, 491, 492, 493, 737, 738, 739],
    'long_beside_short': [40000, 3, 128, 1, 20000, 250, 7],
}


@pytest.mark.parametrize('name', list(LENGTHS))
@pytest.mark.parametrize('MT', [1, 2])
@pytest.mark.parametrize('chain', [False, True])
def test_ragged_single_conv_items_cover_every_live_tile_once(name, MT, chain):
    """The ResBlock layer sets of a merged launch (k 3 / 7 / 11, chain-ordered with the running sum or not)."""
    lengths = LENGTHS[name]
    KS, hr = [3, 7, 11], [1, 1, 1]
    accum = [0, 1, 1] if chain else [0, 0, 0]
    items, off, P, bal = ragged(KS, hr, accum, lengths, MT=MT, chain=chain)
    assert P == 0 and 0 < bal <= 1.0
    check(items, off, 3, lengths, 1, lambda mt: 128 * mt, chain, False)


@pytest.mark.parametrize('name', list(LENGTHS))
@pytest.mark.parametrize('col_blocks', [1, 4])
def test_ragged_single_layer_with_column_blocks(name, col_blocks):
    """One layer over several column blocks (the upsamplers and the C = 256 / 512 convolutions)."""
    lengths = LENGTHS[name]
    items, off, _, _ = ragged([7], [0], [0], lengths, MT=2, col_blocks=col_blocks, Cin=256)
    check(items, off, 1, lengths, col_blocks, lambda mt: 128 * mt, False, False)


@pytest.mark.parametrize('name', list(LENGTHS))
@pytest.mark.parametrize('chain', [False, True])
def test_ragged_fused_items_cover_every_output_row_once(name, chain):
    """Fused ResBlock1 items (stage-3 chains of config 2): P output rows each, none past the clip's end."""
    lengths = LENGTHS[name]
    KS1, KS2 = [3, 7, 11], [3, 7, 11]
    accum = [0, 1, 1] if chain else [0, 0, 0]
    items, off, P, bal = ragged(KS1, [1, 1, 1], accum, lengths, MT=2, chain=chain, KS2=KS2, Cin=32)
    assert P == 246 and 0 < bal <= 1.0
    check(items, off, 3, lengths, 1, lambda mt: P, chain, True)


@pytest.mark.parametrize('B,Tq', [(6, 300), (16, 41 * 256 - 3), (1, 1), (3, 128), (5, 129)])
@pytest.mark.parametrize('MT', [1, 2])
@pytest.mark.parametrize('chain', [False, True])
def test_equal_lengths_reproduce_the_uniform_schedule(B, Tq, MT, chain):
    KS, hr = [3, 7, 11], [1, 1, 1]
    accum = [0, 1, 1] if chain else [0, 0, 0]
    got, off_g, _, _ = ragged(KS, hr, accum, [Tq] * B, MT=MT, chain=chain)
    want, off_w = uniform(KS, hr, accum, B, Tq, MT=MT, chain=chain)
    assert np.array_equal(got[:, :5], want) and np.array_equal(off_g, off_w)
    assert (got[:, 5] == Tq).all()


@pytest.mark.parametrize('B,Tq', [(16, 32768), (1, 256), (3, 5 * 246), (4, 41 * 256 - 3)])
@pytest.mark.parametrize('chain', [False, True])
def test_equal_lengths_reproduce_the_uniform_fused_schedule(B, Tq, chain):
    KS1, dil1, KS2 = [3, 7, 11], [5, 5, 5], [3, 7, 11]
    accum = [0, 1, 1] if chain else [0, 0, 0]
    got, off_g, P, _ = ragged(KS1, [1, 1, 1], accum, [Tq] * B, MT=2, chain=chain, KS2=KS2, Cin=32)
    want, off_w, Pw = uniform_fused(KS1, dil1, KS2, accum, B, Tq, chain)
    assert P == Pw
    assert np.array_equal(got[:, :5], want[:, :5]) and np.array_equal(off_g, off_w)


def test_ragged_probe_rejects_bad_lengths():
    N = _lib()
    for lengths in ([5, 0, 3], [-1]):
        with pytest.raises(RuntimeError):
            ragged([3], [0], [0], lengths)
    with pytest.raises(RuntimeError):                              # fused items are two tiles of one column block
        ragged([3], [1], [0], [300], MT=1, KS2=[3], Cin=32)
    assert N is not None

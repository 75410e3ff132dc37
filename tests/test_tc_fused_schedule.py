"""Host logic of the fused ResBlock1 launches (csrc/conv_tc.cu: tc_schedule with fused items, tc_fused_slab): one item runs
c1 and c2 of one dilation step of one chain for P output rows.  No GPU needed."""
import ctypes

import numpy as np
import pytest

K_MAX_ITEMS = 120


def _fused_schedule(KS1, dil1, KS2, accum, B, Tq, chain_ordered, grid=132, Cin=32):
    from neuralsvb_b200 import _native
    arr = lambda v: np.ascontiguousarray(v, dtype=np.int32)
    k1, d1, k2, ac = arr(KS1), arr(dil1), arr(KS2), arr(accum)
    cap = 200000
    items, off, P, bal = np.zeros((cap, 7), np.int32), np.zeros(grid + 1, np.int32), ctypes.c_int32(), ctypes.c_double()
    cnt = _native.check(_native.lib().svb_tc_fused_schedule_probe(len(KS1), k1.ctypes.data, d1.ctypes.data, k2.ctypes.data, ac.ctypes.data,
                                                                   Cin, B, Tq, int(chain_ordered), grid, items.ctypes.data, cap,
                                                                   off.ctypes.data, ctypes.byref(P), ctypes.byref(bal)),
                        'tc_fused_schedule_probe')
    return items[:cnt], off, P.value, bal.value


def _check(items, off, P, KS1, dil1, KS2, B, Tq):
    n = len(KS1)
    assert P == 256 - 2 * max((k - 1) // 2 for k in KS2)
    assert off[0] == 0 and off[-1] == len(items) and (np.diff(off) >= 0).all()
    assert (np.diff(off) <= K_MAX_ITEMS).all()
    assert (items[:, 1] == 0).all() and (items[:, 4] == 2).all()           # one column block, 256 c1 rows
    # every output row of every (layer, clip) exactly once
    cover = np.zeros((n, B, Tq), np.int32)
    for l, _, b, t0, _, _, _ in items:
        cover[l, b, t0:min(t0 + P, Tq)] += 1
    assert (cover == 1).all()
    in_Tp = (Tq + 255) // 256 * 256 + 128                                   # padded rows of a clip's channel group
    for l, _, b, t0, _, row0, rows in items:
        h1, h2 = (KS1[l] - 1) // 2 * dil1[l], (KS2[l] - 1) // 2
        assert row0 >= 0 and row0 + rows <= in_Tp                            # the copy stays inside the channel group
        assert row0 == 64 + t0 - h2 - h1 and rows <= 256 + 2 * h1
        # the c1 rows that feed kept outputs and lie in [0, Tq) have their whole tap window in the copy
        lo, hi = max(t0 - h2, 0), min(t0 + P + h2, Tq)
        if hi > lo:
            assert row0 <= 64 + lo - h1 and 64 + hi - 1 + h1 < row0 + rows


@pytest.mark.parametrize('B,Tq', [(16, 32768), (1, 256), (1, 512), (1, 768), (1, 37 * 256), (3, 5 * 246), (2, 1000), (4, 41 * 256 - 3)])
@pytest.mark.parametrize('chain', [False, True])
def test_fused_items_cover_every_output_row_once_inside_the_clip(B, Tq, chain):
    """Stage-3 chains of config 2 (k 3 / 7 / 11, dilation 5 step): the bench shape, clips shorter than one item (one mel frame
    = 256 rows), lengths that are not a multiple of P or 256."""
    KS1, dil1, KS2 = [3, 7, 11], [5, 5, 5], [3, 7, 11]
    accum = [0, 1, 1] if chain else [0, 0, 0]
    items, off, P, bal = _fused_schedule(KS1, dil1, KS2, accum, B, Tq, chain)
    assert P == 246
    _check(items, off, P, KS1, dil1, KS2, B, Tq)
    assert 0 < bal <= 1.0


def test_chain_ordered_fused_items_of_a_clip_share_rows():
    """The step that adds the chains into the stage output: every CTA runs chains 0, 1, 2 of the same rows back to back, so the
    read-modify-write of the ResBlock sum stays in one thread."""
    items, off, P, _ = _fused_schedule([3, 7, 11], [1, 1, 1], [3, 7, 11], [0, 1, 1], 16, 16384, True, Cin=64)
    for c in range(len(off) - 1):
        mine = items[off[c]:off[c + 1]]
        assert len(mine) % 3 == 0
        for i in range(0, len(mine), 3):
            assert mine[i:i + 3, 0].tolist() == [0, 1, 2]
            assert (mine[i:i + 3, 1:5] == mine[i, 1:5]).all()


def test_small_c2_halo_widens_the_item():
    """P follows the largest c2 halo of the launch: k 3 only leaves 254 output rows per item."""
    items, off, P, _ = _fused_schedule([3], [3], [3], [0], 2, 3000, False, grid=8)
    assert P == 254
    _check(items, off, P, [3], [3], [3], 2, 3000)


def test_fused_lists_balance_long_and_short_chains():
    """Plain (not chain-ordered) bench-shape list: the k 11 items cost more than the k 3 ones, LPT still balances them."""
    items, off, P, bal = _fused_schedule([3, 7, 11], [3, 3, 3], [3, 7, 11], [0, 0, 0], 16, 16384, False, Cin=64)
    _check(items, off, P, [3, 7, 11], [3, 3, 3], [3, 7, 11], 16, 16384)
    assert bal > 0.95

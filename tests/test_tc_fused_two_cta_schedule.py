"""Host logic of the fused C = 32 ResBlock1 launches at two CTAs per SM (csrc/conv_tc.cu: tc_plan with ctas = 2,
tc_worklist_build): the work lists are built over 2 x 132 = 264 CTAs of an H100.  No GPU needed."""
import numpy as np
import pytest

from tests.test_tc_fused_schedule import K_MAX_ITEMS, _check, _fused_schedule

GRID = 2 * 132
KS = [3, 7, 11]


@pytest.mark.parametrize('dil', [1, 3, 5])
@pytest.mark.parametrize('B,Tq', [(16, 32768), (1, 256), (1, 246), (3, 77 * 256), (2, 41 * 256 - 3), (64, 32768)])
@pytest.mark.parametrize('chain', [False, True])
def test_two_cta_lists_cover_every_output_row_once(dil, B, Tq, chain):
    """Stage 3 of the bench config at each dilation step: the bench shape (16 clips x 128 frames x 256), a clip of one frame, a
    clip shorter than one item, odd lengths, and a batch four times the bench's that still fits the per-CTA item table."""
    accum = [0, 1, 1] if chain else [0, 0, 0]
    items, off, P, bal = _fused_schedule(KS, [dil] * 3, KS, accum, B, Tq, chain, grid=GRID)
    assert len(off) == GRID + 1
    _check(items, off, P, KS, [dil] * 3, KS, B, Tq)
    assert (np.diff(off) <= K_MAX_ITEMS).all()
    assert 0 < bal <= 1.0
    if chain:
        # the running ResBlock sum: chains 0, 1, 2 of the same rows back to back in one CTA, so the order is unchanged
        for c in range(GRID):
            mine = items[off[c]:off[c + 1]]
            assert len(mine) % 3 == 0
            for i in range(0, len(mine), 3):
                assert mine[i:i + 3, 0].tolist() == [0, 1, 2]
                assert (mine[i:i + 3, 1:5] == mine[i, 1:5]).all()


def test_two_cta_lists_balance_the_bench_shape():
    """16 x 32768 rows: 2144 items per chain, about 24 per CTA over 264 CTAs; LPT keeps the load within 5 % of the mean."""
    items, off, P, bal = _fused_schedule(KS, [5] * 3, KS, [0, 0, 0], 16, 32768, False, grid=GRID)
    assert P == 246 and len(items) == 3 * 16 * -(-32768 // 246)
    assert np.diff(off).max() <= 30
    assert bal >= 0.95, bal


def test_two_cta_chain_ordered_list_is_as_even_as_its_units_allow():
    """The step with the running sum schedules whole (chain 0, 1, 2) triples of equal cost: 2144 of them over 264 CTAs is at
    most ceil(2144 / 264) = 9 triples per CTA, a balance of 2144 / 264 / 9."""
    items, off, P, bal = _fused_schedule(KS, [5] * 3, KS, [0, 1, 1], 16, 32768, True, grid=GRID)
    units = 16 * -(-32768 // 246)
    assert np.diff(off).max() == 3 * -(-units // GRID)
    assert bal == pytest.approx(units / GRID / -(-units // GRID))

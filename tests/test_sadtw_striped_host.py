"""The striped shape-aware DTW's planner (svb_sadtw_striped_plan), host only: stripe cover, the memory model, the choice between
single pass and checkpointed, the refusals, and the Python wrappers' checks before any device work.  No GPU needed."""
import ctypes
import os

import numpy as np
import pytest

from neuralsvb_b200 import _native
from neuralsvb_b200.modules.voice_conversion.dtw import core

SINGLE, CHECKPOINTED = 0, 1
SEQ_META, PAIR_META, STRIPE_PAIR, WALK_STATE = 88, 40, 24, 16       # sizeof of the workspace's per-sequence / per-pair records
SINGLE_PASS_DIAGS, MAX_STRIPE_DIAGS = 512, 8192
GiB = 1 << 30


@pytest.fixture(scope='module')
def lib():
    try:
        _native.build()
    except RuntimeError:
        if not os.path.exists(_native.LIB_PATH):
            raise
    return _native.lib()


@pytest.fixture(autouse=True)
def no_hooks(monkeypatch):
    monkeypatch.delenv('SVB_DTW_STRIPE_DIAGS', raising=False)
    monkeypatch.delenv('SVB_DTW_CTA_CELLS', raising=False)


def _arr(v):
    a = np.ascontiguousarray(v, dtype=np.int32)
    return a, ctypes.c_void_p(a.ctypes.data)


def plan(lib, S, T, budget):
    """(status, plan) of svb_sadtw_striped_plan."""
    (sa, sp), (ta, tp) = _arr(S), _arr(T)
    p = core.StripePlan()
    return lib.svb_sadtw_striped_plan(len(S), sp, tp, budget, ctypes.byref(p)), p


def up(x):
    return (x + 255) // 256 * 256


def model(S, T, K, single):
    """The documented memory model: section offsets and total at stripe width K."""
    n = len(S)
    mins = [min(s, t) for s, t in zip(S, T)]
    slots = sum((1 if single else -(-(s + t - 1) // K)) * m for s, t, m in zip(S, T, mins))
    off = [0]
    off.append(up(2 * n * SEQ_META))
    off.append(up(off[1] + n * PAIR_META))
    off.append(up(off[2] + n * STRIPE_PAIR))
    off.append(up(off[3] + (sum(S) + sum(T)) * 48 * 4))
    off.append(up(off[4] + 2 * K * sum(mins) * 4))
    off.append(up(off[5] + (sum(s * t for s, t in zip(S, T)) if single else K * sum(mins))))
    off.append(up(off[6] + slots * 2 * 4))
    return off, up(off[7] + n * WALK_STATE)


def refused(rc, what, lib):
    return rc == -1 and what in lib.svb_last_error()


SHAPES = [([17], [21]), ([2], [2]), ([2, 300, 40], [90, 2, 40]), ([9000, 700, 20000], [8500, 900, 19000]), ([65536], [60000])]


@pytest.mark.parametrize('K', (1, 2, 3, 7, 64, 100, 1024, 40000, 131072))
def test_forced_stripes_cover_every_pair_once(lib, monkeypatch, K):
    monkeypatch.setenv('SVB_DTW_STRIPE_DIAGS', str(K))
    for S, T in SHAPES:
        rc, p = plan(lib, S, T, 1 << 62)
        assert rc == 0 and p.mode == CHECKPOINTED and p.stripe_diags == K
        D = [s + t - 1 for s, t in zip(S, T)]
        assert p.stripes == -(-max(D) // K)
        for d in D:                                 # stripes [k K, (k + 1) K) clipped to [0, D): each diagonal exactly once
            covered = np.zeros(d, np.int32)
            for k in range(p.stripes):
                covered[k * K:min((k + 1) * K, d)] += 1
            assert (covered == 1).all()
        off, total = model(S, T, K, False)
        assert list(p.offsets) == off and p.total_bytes == total


def test_total_is_the_model_and_single_pass_is_chosen_exactly_when_it_fits(lib):
    rs = np.random.RandomState(3)
    for S, T in SHAPES:
        ks = min(SINGLE_PASS_DIAGS, max(s + t - 1 for s, t in zip(S, T)))
        _, single = model(S, T, ks, True)
        rc, p = plan(lib, S, T, single)
        assert rc == 0 and p.mode == SINGLE and p.stripe_diags == ks and p.total_bytes == single
        assert list(p.offsets) == model(S, T, ks, True)[0]
        minimum = p.min_budget_bytes
        extra = list(rs.randint(minimum, single, 5)) if minimum < single else []
        for budget in [single - 1, minimum, (minimum + single) // 2] + extra:
            if budget < minimum:
                continue
            rc, p = plan(lib, S, T, int(budget))
            assert rc == 0 and p.total_bytes <= budget
            if budget < single:
                K = p.stripe_diags
                assert p.mode == CHECKPOINTED and K & (K - 1) == 0 and K <= MAX_STRIPE_DIAGS
                assert p.total_bytes == model(S, T, K, False)[1]
                D = max(s + t - 1 for s, t in zip(S, T))
                assert 2 * K > MAX_STRIPE_DIAGS or K >= D or model(S, T, 2 * K, False)[1] > budget   # the largest that fits
        assert minimum == min([single] + [model(S, T, 1 << e, False)[1] for e in range(14)
                                          if (1 << e) < 2 * max(s + t - 1 for s, t in zip(S, T))])


def test_a_65536_frame_pair_in_one_gib():
    """The worked example: one 65536 x 65536 pair at 1 GiB is checkpointed at K = 1024 with 0.54 GB of stripe cost, 67 MB of
    stripe directions and 67 MB of checkpoints; single pass needs the 4.3 GB of directions."""
    p = core.striped_plan([65536], [65536], GiB)
    assert p.mode == CHECKPOINTED and p.stripe_diags == 1024 and p.stripes == 128
    o = list(p.offsets) + [p.total_bytes]
    assert o[5] - o[4] == 2 * 1024 * 65536 * 4 and o[6] - o[5] == 1024 * 65536 and o[7] - o[6] == 128 * 2 * 65536 * 4
    big = core.striped_plan([65536], [65536], 24 * GiB)
    assert big.mode == SINGLE and big.offsets[6] - big.offsets[5] == 65536 ** 2
    assert core.striped_workspace_bytes([65536], [65536], GiB) == p.total_bytes <= GiB
    assert core.long_workspace_bytes([65536], [65536]) > 5 * 65536 ** 2 > big.total_bytes


def test_refusals_name_their_reason(lib, monkeypatch):
    _, p = plan(lib, [9000], [10000], 1 << 62)
    m = p.min_budget_bytes
    rc, _ = plan(lib, [9000], [10000], m - 1)
    assert refused(rc, f'below the minimum of {m} bytes'.encode(), lib)
    assert plan(lib, [9000], [10000], m)[0] == 0
    assert refused(plan(lib, [65537], [9000], 1 << 62)[0], b'at most 65536', lib)
    assert refused(plan(lib, [9000, 100], [9000, 70000], 1 << 62)[0], b'at most 65536', lib)
    assert refused(plan(lib, [1], [9000], 1 << 62)[0], b'at least 2', lib)
    assert refused(plan(lib, [50, 9000], [50, 1], 1 << 62)[0], b'at least 2', lib)
    (sa, sp), (ta, tp) = _arr([100]), _arr([100])
    assert refused(lib.svb_sadtw_striped_plan(1, sp, tp, 1 << 40, None), b'null argument', lib)
    assert refused(lib.svb_sadtw_striped_plan(1, None, tp, 1 << 40, ctypes.byref(core.StripePlan())), b'null length', lib)
    assert refused(lib.svb_sadtw_striped_plan(0, sp, tp, 1 << 40, ctypes.byref(core.StripePlan())), b'pairs', lib)
    monkeypatch.setenv('SVB_DTW_STRIPE_DIAGS', '8192')           # a forced K whose workspace exceeds the budget
    assert refused(plan(lib, [9000], [10000], m)[0], b'SVB_DTW_STRIPE_DIAGS=8192 needs', lib)
    for bad in ('0', '131073', 'x'):
        monkeypatch.setenv('SVB_DTW_STRIPE_DIAGS', bad)
        assert refused(plan(lib, [9000], [10000], 1 << 40)[0], b'SVB_DTW_STRIPE_DIAGS', lib)


def test_align_striped_refuses_before_any_launch(lib):
    """Host buffers stand in for every device pointer: each refusal must come before the call touches one."""
    buf = np.zeros(1 << 16, np.float64)
    p = ctypes.c_void_p(buf.ctypes.data)
    _, pl = plan(lib, [9000], [10000], 2 * GiB)

    def align(S, T, ws_bytes, budget=2 * GiB, dtype=0, variant=1, alignment=p):
        (sa, sap), (ta, tap) = _arr(S), _arr(T)
        return lib.svb_sadtw_align_striped(p, p, dtype, variant, len(S), sap, tap, None, p, ws_bytes, budget, alignment, None, None,
                                           None)

    assert refused(align([9000], [10000], pl.total_bytes - 1), b'workspace', lib)
    assert refused(align([9000], [10000], pl.total_bytes, budget=1000), b'below the minimum', lib)
    assert refused(align([65537], [10000], 1 << 40), b'at most 65536', lib)
    assert refused(align([9000], [10000], pl.total_bytes, alignment=None), b'null argument', lib)
    assert refused(align([9000], [10000], pl.total_bytes, dtype=2), b'bad f0 dtype', lib)
    assert refused(align([9000], [10000], pl.total_bytes, variant=3), b'bad variant', lib)
    assert (buf == 0).all()


def test_python_wrappers_refuse_before_device_work(lib, monkeypatch):
    def no_device(*a):
        raise AssertionError('device work before the checks')
    monkeypatch.setattr(core, 'device_of', no_device)
    a, b = np.linspace(200.0, 220.0, 9000), np.linspace(200.0, 220.0, 10000)
    with pytest.raises(ValueError, match='below the minimum of [0-9]+ bytes'):
        core.align_songs([a], [b], workspace_bytes=1 << 20)
    with pytest.raises(ValueError, match='at most 65536'):
        core.align_songs([np.ones(65537)], [b])
    with pytest.raises(ValueError, match='at least 2'):
        core.align_songs([np.ones(1)], [b])
    with pytest.raises(ValueError, match=r'\[S\] or \[S, 1\]'):
        core.align_songs([np.ones((9, 2))], [b])
    with pytest.raises(ValueError, match='align_songs runs'):
        core.align_songs([a], [b], 'NaiveDTW')
    with pytest.raises(ValueError, match='1 amateur and 2 professional'):
        core.align_songs([a], [b, b])
    with pytest.raises(ValueError, match='below the minimum'):
        core.striped_workspace_bytes([9000], [10000], 1 << 20)
    assert core.striped_workspace_bytes([9000, 30], [10000, 40], 24 * GiB) <= 24 * GiB

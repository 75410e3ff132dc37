"""Whole songs, host side: plan_song's invariants and refusals, stitch_mels against a numpy restatement, and the C ABI's refusals of
the long-pair DTW before any launch.  No GPU needed."""
import ctypes
import os

import numpy as np
import pytest
import torch

from neuralsvb_b200 import _native
from neuralsvb_b200.inference.song_plan import plan_song, stitch_mels, stitch_weights

HP = {'frames_multiple': 4, 'max_frames': 5000}


def random_song(rs, Tp, Ta):
    """A monotone alignment of Tp professional frames onto Ta amateur ones with local tempo changes, and uv runs."""
    rate = np.exp(rs.normal(0, 0.3, Tp // 200 + 2)).repeat(200)[:Tp]
    pos = np.cumsum(rate)
    a2p = np.minimum((pos / pos[-1] * (Ta - 1)).astype(np.int64), Ta - 1)
    uv = (rs.rand(Tp // 20 + 1) < 0.3).repeat(20)[:Tp].astype(np.float32)
    return a2p, uv


def check_invariants(plan, Tp, Ta, a2p, seg, ov, hp=HP):
    fm, mx = hp['frames_multiple'], hp['max_frames']
    assert plan[0][0] == 0 and plan[-1][1] == Tp
    for k, (s, e, lo, hi) in enumerate(plan):
        assert all(x % fm == 0 for x in (s, e, lo, hi))
        assert 60 <= e - s <= seg and 60 <= hi - lo <= mx and 0 <= lo < hi <= Ta
        assert lo <= a2p[s:e].min() and a2p[s:e].max() < hi
        if k:
            assert s == plan[k - 1][1] - ov and s > plan[k - 1][0]


@pytest.mark.parametrize('seed', range(12))
def test_plan_invariants_on_random_alignments(seed):
    rs = np.random.RandomState(seed)
    Tp = int(rs.randint(5001, 45000)) // 4 * 4
    Ta = int(Tp * rs.uniform(0.85, 1.15)) // 4 * 4
    seg, ov = [(5000, 64), (2000, 32), (1000, 0), (4000, 128)][seed % 4]
    a2p, uv = random_song(rs, Tp, Ta)
    plan = plan_song(Tp, Ta, a2p, uv, HP, seg, ov)
    check_invariants(plan, Tp, Ta, a2p, seg, ov)
    assert len(plan) >= -(-Tp // seg)


def test_one_segment_is_the_whole_cropped_pair():
    rs = np.random.RandomState(0)
    a2p, uv = random_song(rs, 4000, 5000)
    assert plan_song(4000, 5000, a2p, uv, HP) == [(0, 4000, 0, 5000)]
    a2p, uv = random_song(rs, 60, 60)
    assert plan_song(60, 60, a2p, uv, HP) == [(0, 60, 0, 60)]
    # an amateur take over max_frames makes even a short professional take a planned song
    a2p, uv = random_song(rs, 4000, 5200)
    plan = plan_song(4000, 5200, a2p, uv, HP)
    check_invariants(plan, 4000, 5200, a2p, 5000, 64)


def test_a_cut_prefers_the_most_unvoiced_overlap_and_the_latest_on_a_tie():
    Tp, Ta, seg, ov = 2400, 2400, 1000, 64
    a2p = np.arange(Tp)
    uv = np.zeros(Tp)
    uv[800:860] = 1                   # inside the last quarter [750, 1000] of the first window: the overlap [e - 64, e) around it
    plan = plan_song(Tp, Ta, a2p, uv, HP, seg, ov)
    assert plan[0][1] in range(860, 868)                        # every end in 860 .. 864 holds all 60; the latest wins
    assert plan[0][1] == 864
    none = plan_song(Tp, Ta, a2p, np.zeros(Tp), HP, seg, ov)
    assert none[0][1] == 1000                                   # no unvoiced frame anywhere: the latest end
    early = np.zeros(Tp)
    early[100:200] = 1                                          # before the last quarter: not a candidate
    assert plan_song(Tp, Ta, a2p, early, HP, seg, ov)[0][1] == 1000


def test_an_amateur_span_over_max_frames_ends_the_segment_earlier():
    Tp, Ta = 6000, 12000
    a2p = np.minimum(np.arange(Tp) * 2, Ta - 1)                 # two amateur frames per professional frame
    plan = plan_song(Tp, Ta, a2p, np.zeros(Tp), HP)
    check_invariants(plan, Tp, Ta, a2p, 5000, 64)
    assert max(e - s for s, e, _, _ in plan) <= 2500


@pytest.mark.parametrize('case,msg', [
    ('short_prof', 'song 3: cannot plan the segments at professional frame 0: .*fewer than 60'),
    ('short_ama', 'song 3: cannot plan the segments at professional frame 0'),
    ('pile', 'song 3: cannot plan the segments at professional frame 0: every segment end'),
    ('pile_late', 'song 3: cannot plan the segments at professional frame [1-9]'),
    ('uncropped', 'not cropped to a multiple of 4'),
    ('segment', 'segment_frames = 5004'),
    ('overlap', 'overlap_frames = 66'),
    ('overlap_big', 'overlap_frames = 2504'),
    ('align_short', '100 alignment entries'),
    ('align_range', 'outside the 6000 amateur frames'),
])
def test_every_refusal_names_the_song(case, msg):
    Tp, Ta, seg, ov = 6000, 6000, None, 64
    a2p, uv = np.arange(6000), np.zeros(6000)
    if case == 'short_prof':
        Tp = 56
    elif case == 'short_ama':
        Ta, a2p = 56, np.minimum(a2p, 55)
        Tp = 7000
        a2p, uv = np.minimum(np.arange(7000), 55), np.zeros(7000)
    elif case == 'pile':
        Ta, Tp = 20000, 6000
        a2p = np.where(np.arange(Tp) < 60, np.arange(Tp) * 200, 19999).clip(max=19999)
    elif case == 'pile_late':
        Ta, Tp = 20000, 12000
        a2p = np.where(np.arange(Tp) < 8000, np.arange(Tp) // 2, 19999)
        uv = np.zeros(Tp)
    elif case == 'uncropped':
        Tp = 5999
    elif case == 'segment':
        seg = 5004
    elif case == 'overlap':
        ov = 66
    elif case == 'overlap_big':
        seg, ov = 5000, 2504
    elif case == 'align_short':
        Tp, Ta, a2p = 8000, 8000, np.arange(100)
    elif case == 'align_range':
        Tp, a2p, uv = 8000, np.arange(8000), np.zeros(8000)
    with pytest.raises(ValueError, match=msg):
        plan_song(Tp, Ta, a2p, uv, HP, seg, ov, name='song 3')


def test_stitch_equals_the_numpy_restatement():
    rs = np.random.RandomState(3)
    Tp, Ta, ov = 14000, 13000, 64
    a2p, uv = random_song(rs, Tp, Ta)
    plan = plan_song(Tp, Ta, a2p, uv, HP, 5000, ov)
    assert len(plan) >= 3
    mels = [rs.normal(0, 1, (e - s + int(rs.randint(0, 9)), 80)).astype(np.float32) for s, e, _, _ in plan]
    got = stitch_mels([torch.from_numpy(m) for m in mels], plan, ov).numpy()
    w = (np.arange(ov, dtype=np.float32) + np.float32(0.5)) / np.float32(ov)
    assert np.array_equal(w, stitch_weights(ov))
    ref = np.empty((Tp, 80), np.float32)
    for k, (s, e, _, _) in enumerate(plan):
        ref[s:e] = mels[k][:e - s]
    for k in range(len(plan) - 1):
        s0, s1 = plan[k][0], plan[k + 1][0]
        for t in range(s1, s1 + ov):
            wt = np.float32((t - s1 + 0.5) / ov)
            ref[t] = (np.float32(1) - wt) * mels[k][t - s0] + wt * mels[k + 1][t - s1]
    assert got.dtype == np.float32 and np.array_equal(got, ref)
    one = [(0, 400, 0, 400)]
    assert np.array_equal(stitch_mels([torch.from_numpy(mels[0][:400])], one, ov).numpy(), mels[0][:400])


@pytest.fixture(scope='module')
def lib():
    try:
        _native.build()
    except RuntimeError:
        if not os.path.exists(_native.LIB_PATH):
            raise
    return _native.lib()


def _arr(v, dt=np.int32):
    a = np.ascontiguousarray(v, dtype=dt)
    return a, ctypes.c_void_p(a.ctypes.data)


def test_long_c_abi_rejects_before_any_launch(lib, monkeypatch):
    """Host buffers stand in for every device pointer: each refusal must come before the call touches one."""
    buf = np.zeros(1 << 16, np.float64)
    p = ctypes.c_void_p(buf.ctypes.data)

    def size(S, T, fn=lib.svb_sadtw_long_workspace_bytes):
        (sa, sp), (ta, tp) = _arr(S), _arr(T)
        return fn(len(S), sp, tp, None)

    assert size([65536], [65536]) > 65536 ** 2 * 5
    assert size([65537], [100]) == -1 and size([100], [65537]) == -1 and size([9000, 70000], [9000, 9000]) == -1
    assert size([9000], [9000]) > 9000 ** 2 * 5
    assert size([9000], [9000], lib.svb_sadtw_workspace_bytes) == -1          # the one-CTA entry keeps its bound
    assert size([8000, 30], [8000, 40]) == size([8000, 30], [8000, 40], lib.svb_sadtw_workspace_bytes)

    def align(S, T, ws_bytes):
        sa, sap = _arr(S)
        ta, tap = _arr(T)
        return lib.svb_sadtw_align_long(p, p, 0, 1, len(S), sap, tap, None, p, ws_bytes, p, None, None, None)

    def refused(rc, what):
        return rc == -1 and what in lib.svb_last_error()

    assert refused(align([65537], [9000], 1 << 40), b'at most 65536')
    assert refused(align([9000], [66000], 1 << 40), b'at most 65536')
    need = size([9000], [10000])
    assert refused(align([9000], [10000], need - 1), b'workspace')
    for bad in ('0', '8193', 'x'):
        monkeypatch.setenv('SVB_DTW_CTA_CELLS', bad)
        assert refused(align([9000], [10000], need), b'SVB_DTW_CTA_CELLS')
    assert (buf == 0).all()


def test_beautify_songs_refuses_bad_segments_before_device_work_and_unplannable_songs_before_the_model():
    """The beautifier's host code with fake device stages (tests/test_beautify_host.py): bad segment arguments raise before the
    front end; a song whose alignment piles more than max_frames amateur frames onto its first window raises naming the song and
    frame after the alignment, before the model."""
    from neuralsvb_b200.utils import hparams as H
    from tests.test_beautify_host import EMB, FakeBeautifier, take
    saved = dict(H.hparams)
    H.hparams.clear()
    H.hparams.update({'audio_sample_rate': 22050, 'hop_size': 128, 'max_frames': 5000, 'frames_multiple': 4, 'pitch_norm': 'standard',
                      'use_uv': True, 'f0_mean': 300.0, 'f0_std': 80.0, 'latent_size': 128, 'disable_map': False,
                      'vocoder_denoise_c': 0.0})
    try:
        class Fake(FakeBeautifier):
            def _align_songs(self, f0_dev, frames, st):
                self.calls.append('align')
                B = len(frames) // 2
                return [np.where(np.arange(frames[B + i]) < 100, 0, frames[i] - 1) for i in range(B)]

            def _model_on(self, *a):
                self.calls.append('model')

        b = Fake(H.hparams)
        with pytest.raises(ValueError, match='beautify_songs: overlap_frames = 66'):
            b._run_songs([take(6000, 1)], [take(6000, 2)], [EMB], 1, None, None, 66)
        with pytest.raises(ValueError, match='beautify_songs: segment_frames = 40'):
            b._run_songs([take(6000, 1)], [take(6000, 2)], [EMB], 1, None, 40, 0)
        assert b.calls == []
        with pytest.raises(ValueError, match='song 1: cannot plan the segments at professional frame 0: every segment end'):
            b._run_songs([take(300, 1), take(6000, 3)], [take(300, 2), take(6000, 4)], [EMB, EMB], 1, None, None, 64)
        assert b.calls == ['front_end', 'pitch', 'align']
    finally:
        H.hparams.clear()
        H.hparams.update(saved)

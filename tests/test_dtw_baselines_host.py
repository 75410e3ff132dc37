"""Baseline pitch alignments, host side: the oracle (oracle/dtw_baselines.py) against tests/golden/dtw_baselines.npz, written from
the unmodified reference by oracle/gen_golden_dtw_baselines.py; the f0 round trip; the C ABI's and the Python layer's refusals
before any launch.  No GPU needed."""
import ctypes
import os

import numpy as np
import pytest
import torch

from neuralsvb_b200 import _native
from neuralsvb_b200.modules.voice_conversion.dtw import core
from neuralsvb_b200.modules.voice_conversion.dtw import naive_dtw as ND
from neuralsvb_b200.modules.voice_conversion.dtw import naive_interpo as NI
from neuralsvb_b200.utils import pitch_utils as PU
from neuralsvb_b200.utils import synthetic as S
from oracle import dtw_baselines as O
from oracle import sadtw as OS
from oracle.gen_golden_dtw_baselines import (DTW_METHODS, INTERPO_CASES, KINDS, MATRIX_CASE, MATRIX_CASE_MM, ROUND_TRIPS,
                                             make_input, mel_pair)
from oracle.gen_golden_sadtw import SADTW_CASES

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'dtw_baselines.npz')


@pytest.fixture(scope='module')
def golden():
    return np.load(GOLDEN)


def test_oracle_reproduces_every_reference_alignment(golden):
    for name, (seed, Sn, Tn) in SADTW_CASES.items():
        src, tgt = S.make_f0_pair(seed, Sn, Tn)
        for method in DTW_METHODS:
            for kind in KINDS[method]:
                mine, _ = O.align(method, make_input(kind, src, method), make_input(kind, tgt, method))
                assert np.array_equal(mine, golden[f'{name}/{method}/{kind}/alignment']), (name, method, kind)
    a, b = mel_pair()
    assert np.array_equal(O.align('NaiveDTW', a, b)[0], golden['mel/alignment'])


def test_oracle_cost_and_dtw_matrices(golden):
    for name in (MATRIX_CASE, MATRIX_CASE_MM):
        seed, Sn, Tn = SADTW_CASES[name]
        src, tgt = S.make_f0_pair(seed, Sn, Tn)
        for method in DTW_METHODS:
            for kind in KINDS[method]:
                key = f'{name}/{method}/{kind}'
                c = O.cost(method, make_input(kind, src, method), make_input(kind, tgt, method))
                ref = golden[f'{key}/cost']
                tol = 1e-12 if ref.dtype == np.float64 else 1e-6
                assert c.dtype == ref.dtype and c.shape == (Tn, Sn), key
                assert np.abs(c - ref).max() <= tol * np.abs(ref).max(), key
                d = OS.time_warp(ref)
                assert np.array_equal(d, golden[f'{key}/dtw']), key


def test_nearest_index_matches_interpolate(golden):
    for name, (Sn, Tn) in {**{k: v[1:] for k, v in SADTW_CASES.items()}, **INTERPO_CASES}.items():
        assert golden[f'ninterpo/{name}/params'].tolist() == [Sn, Tn]
        assert np.array_equal(O.nearest_index(Sn, Tn), golden[f'ninterpo/{name}/index']), name
    # the float32 scale matters: exact rational arithmetic picks another frame somewhere on these lengths
    for name, (Sn, Tn) in (('s5000_t4999', (5000, 4999)), ('s4321_t5000', (4321, 5000))):
        exact = np.minimum((np.arange(Tn) * Sn) // Tn, Sn - 1)
        assert not np.array_equal(exact, golden[f'ninterpo/{name}/index']), name


def test_accuracy_matches_job(golden):
    for name, (seed, Sn, Tn) in SADTW_CASES.items():
        m_src, m_tgt = S.make_mel2ph_pair(seed, Sn, Tn)
        assert np.array_equal(m_src, golden[f'{name}/mel2ph_src']) and np.array_equal(m_tgt, golden[f'{name}/mel2ph_tgt'])
        for method in DTW_METHODS:
            for kind in KINDS[method]:
                key = f'{name}/{method}/{kind}'
                acc = O.alignment_accuracy(golden[f'{key}/alignment'], m_src, m_tgt)
                assert acc == golden[f'{key}/accuracy'], key


def test_mel2ph_pair_is_monotone_runs():
    a, b = S.make_mel2ph_pair(21, 1378, 1400)
    for m in (a, b):
        v = m[m > 0]
        assert m.dtype == np.int64 and (np.diff(v) >= 0).all() and v[0] == 1 and (np.diff(v) <= 1).all()
        nz = np.nonzero(m == 0)[0]
        assert len(nz) == 0 or nz[0] == len(v)             # padding only at the end
    assert a.max() == b.max()                             # the same phonemes in both takes


def test_f0_round_trip(golden):
    for norm, hp in ROUND_TRIPS.items():
        for name in ('s60_t48', 's8s'):
            seed, Sn, Tn = SADTW_CASES[name]
            f0 = S.make_f0_pair(seed, Sn, Tn)[0]
            pad = torch.from_numpy(S.make_mel2ph_pair(seed, Sn, Tn)[0]) == 0
            f, uv = PU.norm_interp_f0(f0, hp)
            got = PU.denorm_f0(f, uv, hp, pitch_padding=pad).numpy()
            assert np.array_equal(got, golden[f'roundtrip/{norm}/{name}']), (norm, name)


# ---- the C ABI refuses before touching any pointer: host buffers stand in for device memory ----------------------------------

def _lib():
    _native.build()
    return _native.lib()


def _call(lib, method=0, dtype=0, n=1, S=(40,), T=(50,), H=1, ws_bytes=None, null=None):
    s = np.asarray(S, np.int32)
    t = np.asarray(T, np.int32)
    buf = np.zeros(1 << 16, np.float64)
    out = np.zeros(1 << 12, np.int64)
    p = lambda a: ctypes.c_void_p(a.ctypes.data)  # noqa: E731
    args = dict(src=p(buf), tgt=p(buf), ws=p(buf), out=p(out))
    if null:
        args[null] = None
    need = lib.svb_dtw_baselines_workspace_bytes(method, dtype, n, p(s), p(t))
    wb = (need if need > 0 else 1 << 19) if ws_bytes is None else ws_bytes
    return lib.svb_dtw_baselines_align(args['src'], args['tgt'], dtype, method, n, p(s), p(t), H, args['ws'], wb, args['out'], None,
                                       None, None), lib.svb_last_error().decode()


@pytest.mark.parametrize('kw, msg', [
    (dict(dtype=2), 'bad dtype'),
    (dict(method=5), 'bad method'),
    (dict(method=-1), 'bad method'),
    (dict(method=0, H=2), 'feat_dim'),
    (dict(method=1, H=0), 'feat_dim'),
    (dict(method=1, H=5000), 'feat_dim'),
    (dict(S=(1,)), 'at least 2'),
    (dict(T=(1,)), 'at least 2'),
    (dict(n=0, S=(), T=()), 'pairs'),
    (dict(ws_bytes=16), 'workspace'),
    (dict(null='src'), 'null'),
    (dict(null='tgt'), 'null'),
    (dict(null='ws'), 'null'),
    (dict(null='out'), 'null'),
    (dict(S=(9000,), T=(9000,)), 'anti-diagonal'),
])
def test_abi_refuses_before_launch(kw, msg):
    rc, err = _call(_lib(), **kw)
    assert rc == -1 and msg in err, (rc, err)


def test_abi_cost_entry_refuses():
    lib = _lib()
    buf = np.zeros(1 << 16, np.float64)
    s, t = np.asarray([40], np.int32), np.asarray([50], np.int32)
    p = lambda a: ctypes.c_void_p(a.ctypes.data)  # noqa: E731
    rc = lib.svb_dtw_baselines_cost(p(buf), p(buf), 0, 4, 1, p(s), p(t), 1, p(buf), 1 << 19, p(buf), None)
    assert rc == -1 and 'NInterpo' in lib.svb_last_error().decode()
    rc = lib.svb_dtw_baselines_cost(p(buf), p(buf), 0, 0, 1, p(s), p(t), 1, p(buf), 1 << 19, None, None)
    assert rc == -1 and 'null' in lib.svb_last_error().decode()
    rc = lib.svb_dtw_baselines_cost(p(buf), p(buf), 0, 0, 1, p(s), p(t), 1, p(buf), 64, p(buf), None)
    assert rc == -1 and 'workspace' in lib.svb_last_error().decode()
    assert lib.svb_dtw_baselines_workspace_bytes(0, 0, 1, p(np.asarray([1], np.int32)), p(t)) == -1
    # NInterpo runs no DTW, so no anti-diagonal limit
    big = np.asarray([9000], np.int32)
    assert lib.svb_dtw_baselines_workspace_bytes(4, 0, 1, p(big), p(big)) > 0
    assert lib.svb_abi_version() == 1


# ---- the Python layer raises ValueError / TypeError before looking for a device -------------------------------------------------

def test_python_refusals_come_first():
    f = np.linspace(100, 200, 40)
    with pytest.raises(ValueError, match='method'):
        core.align_batch([f], [f], 'DTW')
    with pytest.raises(ValueError, match='method'):
        core.align_pitch([f], [f], method='nope')
    with pytest.raises(TypeError):
        core.align_batch([f.astype(np.int64)], [f.astype(np.int64)], 'LoNDTW')
    with pytest.raises(TypeError, match='mix'):
        core.align_batch([f, f.astype(np.float32)], [f, f], 'ZMNaiveDTW')
    with pytest.raises(TypeError, match='same type'):
        core.align_batch([f], [f.astype(np.float32)], 'NNaiveDTW')
    with pytest.raises(ValueError, match='at least 2'):
        core.align_batch([f[:1]], [f], 'LoNDTW')
    with pytest.raises(ValueError, match=r'\[S\] or \[S, 1\]'):
        core.align_batch([np.zeros((40, 3))], [np.zeros((40, 3))], 'LoNDTW')
    with pytest.raises(ValueError, match='widths'):
        core.align_batch([np.zeros((40, 3)), np.zeros((40, 4))], [np.zeros((40, 3))] * 2, 'NaiveDTW')
    with pytest.raises(ValueError, match='professional'):
        core.align_batch([np.zeros((40, 3))], [np.zeros((40, 4))], 'NaiveDTW')
    with pytest.raises(ValueError, match='no cost'):
        core.baseline_costs([f], [f], 'NInterpo')
    with pytest.raises(TypeError, match='torch'):
        ND.NaiveDTW(f[:, None], f[:, None], f)
    with pytest.raises(ValueError, match=r'\[S, H\]'):
        ND.NaiveDTW(torch.from_numpy(f), torch.from_numpy(f), f)
    with pytest.raises(TypeError, match='torch'):
        ND.ZMNaiveDTW(f, f, f)
    with pytest.raises(ValueError, match='1-D'):
        ND.NNaiveDTW(torch.from_numpy(f)[:, None], torch.from_numpy(f)[:, None], f)
    with pytest.raises(TypeError, match='torch'):
        NI.NInterpo(f, f, f, np.arange(40))
    with pytest.raises(ValueError, match='alignments'):
        core.alignment_accuracy([np.zeros(4, np.int64)], [], [])
    with pytest.raises(ValueError, match='professional frames'):
        core.alignment_accuracy([np.zeros(4, np.int64)], [np.ones(5, np.int64)], [np.ones(3, np.int64)])
    with pytest.raises(TypeError, match='integers'):
        core.alignment_accuracy([np.zeros(3)], [np.ones(5, np.int64)], [np.ones(3, np.int64)])

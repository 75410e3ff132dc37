"""Shape-aware DTW, host side: the oracle (oracle/sadtw.py) against tests/golden/sadtw.npz, written from the unmodified reference
by oracle/gen_golden_sadtw.py, and the C ABI's refusals before any launch.  No GPU needed."""
import ctypes
import os

import numpy as np
import pytest
import torch

from neuralsvb_b200 import _native
from neuralsvb_b200.utils import synthetic as S
from oracle import sadtw as O
from oracle.gen_golden_sadtw import KINDS, METHODS, SADTW_CASES, make_input

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'sadtw.npz')


@pytest.fixture(scope='module')
def golden():
    return np.load(GOLDEN)


def _pair(name, kind):
    seed, Sn, Tn = SADTW_CASES[name]
    src, tgt = S.make_f0_pair(seed, Sn, Tn)
    return make_input(kind, src), make_input(kind, tgt), Sn, Tn


def test_inputs_regenerate_from_seeds(golden):
    for name, (seed, Sn, Tn) in SADTW_CASES.items():
        assert golden[f'{name}/params'].tolist() == [seed, Sn, Tn]
        a, b = S.make_f0_pair(seed, Sn, Tn)
        a2, b2 = S.make_f0_pair(seed, Sn, Tn)
        assert a.shape == (Sn,) and b.shape == (Tn,) and a.dtype == np.float64
        assert np.array_equal(a, a2) and np.array_equal(b, b2)
        assert np.isfinite(a).all() and np.isfinite(b).all() and (a >= 0).all()
    a, b = S.make_f0_pair(21, 1378, 1400)
    assert (a == 0).any() and (a > 0).mean() > 0.7                      # unvoiced gaps, mostly voiced


@pytest.mark.parametrize('method', METHODS)
@pytest.mark.parametrize('kind', KINDS)
def test_oracle_histograms_are_the_reference(golden, method, kind):
    n = 0
    for name in SADTW_CASES:
        key = f'{name}/{method}/{kind}'
        if f'{key}/hist_src' not in golden:
            continue
        a, b, Sn, Tn = _pair(name, kind)
        assert np.array_equal(O.histogram(a, method), golden[f'{key}/hist_src']), key
        assert np.array_equal(O.histogram(b, method, Tn / Sn), golden[f'{key}/hist_tgt']), key
        n += 1
    assert n >= 8


@pytest.mark.parametrize('method', METHODS)
@pytest.mark.parametrize('kind', KINDS)
def test_oracle_alignments_are_the_reference(golden, method, kind):
    for name in SADTW_CASES:
        if name == 's8s':
            continue                                                    # the 8 s pair: tests/test_gpu_sadtw.py
        a, b, _, _ = _pair(name, kind)
        al, _ = O.shape_aware_align(a, b, method)
        assert np.array_equal(al, golden[f'{name}/{method}/{kind}/alignment']), name


def test_oracle_aligns_the_8s_pair(golden):
    a, b, _, _ = _pair('s8s', 'np32')
    al, _ = O.shape_aware_align(a, b, 'EHSADTW')
    assert np.array_equal(al, golden['s8s/EHSADTW/np32/alignment'])


def test_oracle_cost_and_time_warp_on_the_reference_matrix(golden):
    name, method, kind = golden['matrix/case'].tolist()
    a, b, Sn, Tn = _pair(name, kind)
    ref_cost = golden['matrix/cost']
    _, _, m = O.shape_aware_align(a, b, method, full=True)
    assert m['cost'].shape == ref_cost.shape == (Tn, Sn) and m['cost'].dtype == np.float32
    rel = np.abs(m['cost'].astype(np.float64) - ref_cost) / np.abs(ref_cost).max()
    assert rel.max() < 1e-6, rel.max()
    dtw = O.time_warp(ref_cost)                                        # on the reference's own cost: bit-identical
    assert dtw.dtype == np.float32 and np.array_equal(dtw, golden['matrix/dtw'])
    assert O.align_from_distances(ref_cost) == golden['matrix/alignment'].tolist()


def test_oracle_time_warp_tie_order_and_float64():
    c = np.ones((4, 5))                                                 # every path ties: the first minimum (up) wins
    dtw = O.time_warp(c)
    assert dtw.dtype == np.float64 and dtw[0, 0] == 0 and np.isinf(dtw[0, 1:]).all() and np.isinf(dtw[1:, 0]).all()
    assert O.align_from_dtw(dtw) == [0, 1, 2, 3]
    assert O.align_from_distances(np.ones((1, 3))) == [0] and O.align_from_distances(np.ones((3, 1))) == [0, 0, 0]


def test_short_and_empty_window_contours_raise_value_error():
    with pytest.raises(ValueError):
        O.shape_aware_align(np.array([200.0]), np.array([200.0, 201.0]))
    # scale 0.01: every scaled boundary truncates to 0, so no frame has a neighbour
    with pytest.raises(ValueError):
        O.histogram(np.linspace(200, 210, 5), 'SADTW', 0.01)


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


def test_c_abi_rejects_bad_input_before_any_launch(lib):
    """Host buffers stand in for every device pointer: each call must refuse before it touches one."""
    buf = np.zeros(1 << 20, np.float64)
    p = ctypes.c_void_p(buf.ctypes.data)
    s, sp = _arr([17, 20])
    t, tp = _arr([21, 2])
    off = (ctypes.c_int64 * 5)()
    ws = lib.svb_sadtw_workspace_bytes(2, sp, tp, off)
    cells = 17 * 21 + 20 * 2
    assert ws > 0 and list(off) == sorted(off) and ws - off[4] >= cells and off[4] - off[3] >= 4 * cells
    assert off[3] - off[2] >= 4 * 48 * (37 + 23)

    def align(S, T, dtype=0, variant=1, ws_bytes=ws, scale=None, alignment=p):
        sa, sap = _arr(S)
        ta, tap = _arr(T)
        sca = None if scale is None else _arr(scale, np.float64)
        return lib.svb_sadtw_align(p, p, dtype, variant, len(S), sap, tap, None if sca is None else sca[1], p, ws_bytes, alignment,
                                   None, None, None)

    def refused(rc, what):
        return rc == -1 and what in lib.svb_last_error()

    assert refused(align([17, 20], [21, 2], alignment=None), b'null argument')
    assert refused(align([17, 20], [21, 2], dtype=2), b'bad f0 dtype')
    assert refused(align([17, 20], [21, 2], variant=2), b'bad variant')
    assert refused(align([17, 1], [21, 2]), b'at least 2')
    assert refused(align([17, 20], [21, 0]), b'at least 2')
    assert refused(align([17, 20], [21, 2], ws_bytes=ws - 1), b'workspace')
    assert refused(align([17, 20], [21, 2], scale=[1.0, -1.0]), b'bad scale')
    assert refused(align([17, 20], [21, 2], scale=[1.0, 0.01]), b'no neighbour')
    assert refused(align([9000], [9000], ws_bytes=1 << 40), b'anti-diagonal')
    assert lib.svb_sadtw_workspace_bytes(0, sp, tp, None) == -1
    one, onep = _arr([1])
    assert lib.svb_sadtw_workspace_bytes(1, onep, tp, None) == -1
    # the histogram and cost kernels alone, and time_warp on an arbitrary cost
    hw = lib.svb_sadtw_histogram_workspace_bytes(2)
    assert hw > 0 and lib.svb_sadtw_histogram_workspace_bytes(0) == -1
    sca, sc = _arr([1.0, 0.01], np.float64)
    assert refused(lib.svb_sadtw_histogram(p, 0, 0, 2, sp, sc, p, hw, p, None, None), b'no neighbour')
    assert refused(lib.svb_sadtw_histogram(p, 0, 0, 2, sp, None, p, hw - 1, p, None, None), b'workspace')
    assert refused(lib.svb_sadtw_histogram(p, 0, 5, 2, sp, None, p, hw, p, None, None), b'bad variant')
    assert refused(lib.svb_sadtw_cost(p, 0, p, 4, p, None), b'empty histogram')
    assert refused(lib.svb_sadtw_cost(ctypes.c_void_p(buf.ctypes.data + 4), 3, p, 4, p, None), b'16-byte aligned')
    dw = lib.svb_dtw_workspace_bytes(1, 30, 40)
    assert dw >= 30 * 40 * 9 and lib.svb_dtw_workspace_bytes(2, 30, 40) == -1 and lib.svb_dtw_workspace_bytes(0, 9000, 9000) == -1
    assert refused(lib.svb_dtw_align(p, 1, 30, 40, p, dw - 1, p, None, None, None), b'workspace')
    assert refused(lib.svb_dtw_align(p, 0, 0, 40, p, dw, p, None, None, None), b'empty cost')
    assert refused(lib.svb_dtw_align(None, 0, 30, 40, p, dw, p, None, None, None), b'null argument')
    assert (buf == 0).all()


def test_python_layer_rejects_before_any_launch():
    """The drop-in refuses short, non-finite and mixed-type contours with ValueError / TypeError before it looks for a device."""
    from neuralsvb_b200.modules.voice_conversion.dtw import core
    dev = torch.device('cpu')
    with pytest.raises(ValueError, match='at least 2'):
        core._batch_f0([np.array([200.0])], dev, 'amateur')
    with pytest.raises(ValueError, match='NaN or inf'):
        core._batch_f0([np.array([200.0, np.nan, 3.0])], dev, 'amateur')
    with pytest.raises(TypeError, match='mix'):
        core._batch_f0([np.zeros(3, np.float32), np.zeros(3)], dev, 'amateur')
    with pytest.raises(TypeError):
        core.f0_tensor(np.zeros(3, np.int64), dev)
    from neuralsvb_b200.modules.voice_conversion.dtw import align, shape_aware_dtw
    with pytest.raises(NotImplementedError):
        align.align_from_distances(np.ones((3, 3)), debug=True)
    with pytest.raises(NotImplementedError):
        shape_aware_dtw.f0_to_figure(np.ones(3))
    with pytest.raises(NotImplementedError):
        shape_aware_dtw.cal_hist_of_f0(np.ones(3), max_window=32)

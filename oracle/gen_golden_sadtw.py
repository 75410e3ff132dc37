"""ORACLE tooling (test infrastructure only; see oracle/__init__.py): writes tests/golden/sadtw.npz from the UNMODIFIED reference
shape-aware DTW (modules/voice_conversion/dtw/shape_aware_dtw.py: SADTW, enhance_sadtw.py: EHSADTW, align.py).

    NEURALSVB_REFERENCE=/path/to/NeuralSVB python -m oracle.gen_golden_sadtw

Stubs installed before the import, none of which touches the arithmetic: matplotlib (plotting only), numba.jit as the identity
(time_warp then runs as plain Python on numpy scalars, in the cost's float32), tasks.singing.neural_svb_task (a dataset class the
modules import for their __main__ blocks).  The f0 contours are never stored: synthetic.make_f0_pair regenerates them from the
seeds.  Per case: every alignment; the two histograms for the cases up to 64 frames; the cost and DTW matrices of one small case.
The script fails when oracle/sadtw.py does not reproduce a reference alignment or histogram.
"""
import os
import sys
import types

import numpy as np
import torch

from neuralsvb_b200.utils import synthetic as S
from oracle import ref_harness as R
from oracle import sadtw as O
from oracle.gen_golden import OUT

# name: (seed, S amateur frames, T professional frames)
SADTW_CASES = {
    's2_t2': (11, 2, 2),
    's3_t3': (12, 3, 3),
    's2_t3': (13, 2, 3),
    's17_t2': (14, 17, 2),
    's17_t17': (15, 17, 17),
    's17_t14': (16, 17, 14),
    's17_t21': (17, 17, 21),
    's60_t48': (18, 60, 48),
    's60_t60': (19, 60, 60),
    's48_t60': (20, 48, 60),
    's8s': (21, 1378, 1400),               # an 8 s pair at 22050 Hz / hop 128
}
METHODS = ('SADTW', 'EHSADTW')
KINDS = ('np64', 'np32', 'torch32')
HIST_MAX_FRAMES = 64
MATRIX_CASE = ('s17_t21', 'EHSADTW', 'np32')


def make_input(kind, f):
    if kind == 'np64':
        return f.astype(np.float64)
    if kind == 'np32':
        return f.astype(np.float32)
    return torch.from_numpy(f.astype(np.float32))


def install_stubs():
    R.install()
    mpl = types.ModuleType('matplotlib')
    mpl.use = lambda *a, **k: None
    mpl.pyplot = types.ModuleType('matplotlib.pyplot')
    sys.modules['matplotlib'], sys.modules['matplotlib.pyplot'] = mpl, mpl.pyplot
    numba = types.ModuleType('numba')
    numba.jit = lambda f=None, **k: f if f is not None else (lambda g: g)
    sys.modules['numba'] = numba
    for name in ('tasks', 'tasks.singing'):
        m = types.ModuleType(name)
        m.__path__ = []
        sys.modules[name] = m
    nst = types.ModuleType('tasks.singing.neural_svb_task')
    nst.FastSingingDataset = object
    sys.modules['tasks.singing.neural_svb_task'] = nst


def gen_sadtw():
    install_stubs()
    from modules.voice_conversion.dtw import align as ref_align
    from modules.voice_conversion.dtw import enhance_sadtw as ref_eh
    from modules.voice_conversion.dtw import shape_aware_dtw as ref_sa
    ref = {'SADTW': ref_sa, 'EHSADTW': ref_eh}
    out = {}
    for name, (seed, Sn, Tn) in SADTW_CASES.items():
        src, tgt = S.make_f0_pair(seed, Sn, Tn)
        out[f'{name}/params'] = np.array([seed, Sn, Tn], np.int64)
        for method in METHODS:
            for kind in KINDS:
                a, b = make_input(kind, src), make_input(kind, tgt)
                key = f'{name}/{method}/{kind}'
                _, alignment = getattr(ref[method], method)(a, b, a)
                alignment = np.asarray(alignment, np.int64)
                out[f'{key}/alignment'] = alignment
                mine, _ = O.shape_aware_align(a, b, method)
                assert np.array_equal(mine, alignment), f'{key}: the oracle alignment differs from the reference'
                if max(Sn, Tn) <= HIST_MAX_FRAMES:
                    hs = torch.tensor(ref[method].cal_hist_of_f0(a, normalize_hist=True)).numpy()
                    ht = torch.tensor(ref[method].cal_hist_of_f0(b, normalize_hist=True, scale_factor=Tn / Sn)).numpy()
                    assert hs.dtype == np.float32 and ht.dtype == np.float32
                    assert np.array_equal(O.histogram(a, method), hs), f'{key}: amateur histogram'
                    assert np.array_equal(O.histogram(b, method, Tn / Sn), ht), f'{key}: professional histogram'
                    out[f'{key}/hist_src'], out[f'{key}/hist_tgt'] = hs, ht
                if (name, method, kind) == MATRIX_CASE:
                    costs = ref[method].cal_shape_dist(a, b, Sn, Tn).squeeze(0).T.contiguous().numpy()
                    out['matrix/cost'] = costs
                    out['matrix/dtw'] = ref_align.time_warp(costs)
                    out['matrix/alignment'] = np.asarray(ref_align.align_from_distances(costs), np.int64)
                    out['matrix/case'] = np.array(MATRIX_CASE)
                print(key, 'ok', flush=True)
    np.savez_compressed(os.path.join(OUT, 'sadtw.npz'), **out)
    print('sadtw.npz', os.path.getsize(os.path.join(OUT, 'sadtw.npz')), 'bytes')


def main():
    if not R.available():
        sys.exit('gen_golden_sadtw needs NEURALSVB_REFERENCE = a checkout of the reference NeuralSVB')
    os.makedirs(OUT, exist_ok=True)
    gen_sadtw()


if __name__ == '__main__':
    main()
